"""Wall time of `core.evaluation.evaluate_results` for each of the study's four evaluation types on a synthetic
result folder of the study's size: 100 models x 4 case studies x 2 datasets, every approach of Table 1 with its scores,
CAM orders and time files (`--inputs` test inputs per dataset), and every active-learning pickle.  Host only: no GPU
is involved in the evaluation phase.

    python tools/evaluation_bench.py [--inputs 1000] [--repeats 2]
"""
import argparse
import json
import os
import pickle
import sys
import tempfile
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from simple_tip_b200.core import evaluation as E  # noqa: E402
from simple_tip_b200.core import results as R     # noqa: E402

NUM_MODELS = 100


def write_folder(out: str, n: int, seed: int = 0) -> None:
    rng = np.random.default_rng(seed)

    def acc():
        return {(ds, part): int(rng.integers(0, 1000)) / 1000 for ds in E.SPLITS for part in ("observed", "future")}

    for cs in R.CASE_STUDIES:
        for model_id in range(NUM_MODELS):
            R.persist_active_learning(out, cs, model_id, "original", "na", acc())
            for ds in E.SPLITS:
                R.persist(out, cs, ds, "is_misclassified", model_id, rng.random(n) < 0.2)
                for q in R.UNCERTAINTY_APPROACHES:
                    if q == "VR" and cs == "cifar10":
                        continue
                    R.persist(out, cs, ds, f"uncertainty_{q}", model_id, rng.random(n))
                    R.persist_times(out, cs, ds, model_id, q, [0.0, 1.0, 0.1, 0.0])
                for metric in R.COVERAGE_APPROACHES + R.SURPRISE_APPROACHES:
                    R.persist_tip(out, cs, ds, model_id, metric, rng.integers(0, 50, n).astype(np.float64),
                                  cam_order=rng.permutation(n), times=[1.0, 1.0, 1.0, 1.0])
                for approach in R.APPROACHES + ["random"]:
                    if approach == "VR" and cs == "cifar10":
                        continue
                    R.persist_active_learning(out, cs, model_id, approach, ds, acc())


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--inputs", type=int, default=1000, help="test inputs per dataset")
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import pandas  # noqa: F401  (its first import is not the evaluation's)

    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        write_folder(tmp, args.inputs)
        res = {"inputs": args.inputs, "write_folder_s": round(time.perf_counter() - t0, 2)}
        for eval_type in E.EVAL_TYPES:
            times = []
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    E.evaluate_results(tmp, eval_type)
                times.append(round(time.perf_counter() - t0, 3))
            res[eval_type] = times
    print(json.dumps(res))


if __name__ == "__main__":
    main()
