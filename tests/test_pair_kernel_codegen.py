"""What ptxas makes of the tensor-core pass (pair_tc.cu), compiled for sm_90a without a GPU.

ptxas silently serialises wgmma when it cannot keep them asynchronous: it reports C7510 / C7512 / C7520 and
waits for every HGMMA before the next one (`WARPGROUP.DEPBAR` after each).  The DSA filter (`MODE_NN`) hit this
through its candidate staging; in the resident-query variant (the D <= 128 filter) the consumers now only record
events and the drain warps stage them.  This test fails on any such report for a resident-query `pair_kernel`, on
any spill of `pair_kernel`, and checks in the SASS of both resident `MODE_NN` instantiations that no
`WARPGROUP.DEPBAR` separates two HGMMAs.  The streaming variant waits for each K chunk anyway and still stages in
its consumers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "simple_tip_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
if not os.path.exists(NVCC):
    NVCC = shutil.which("nvcc") or NVCC
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="needs nvcc")

# pair_kernel<MODE, EXCL, RESA, F16>: every resident-query instantiation, and the two of MODE_NN
RESIDENT = re.compile(r"_ZN3tip11pair_kernelILi\dELb[01]ELb1ELb[01]E")
NN_KERNELS = [f"_ZN3tip11pair_kernelILi0ELb{excl}ELb1ELb0EEEv14CUtensorMap_stS1_NS_8PairArgsE" for excl in (0, 1)]


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("pair_tc")
    obj = str(out / "pair_tc.o")
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
                          "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, "pair_tc.cu"), "-o", obj],
                         cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return obj, res.stderr


def test_no_serialised_wgmma_or_spills(compiled):
    _, log = compiled
    bad = [l for l in log.splitlines() if re.search(r"\(C75(10|12|20)\)", l) and RESIDENT.search(l)]
    assert not bad, "\n".join(bad)
    # per entry function: "Compiling entry function 'NAME'" ... "N bytes spill stores, M bytes spill loads"
    spills, fn = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn and "pair_kernel" in fn:
            spills[fn] = (int(m.group(1)), int(m.group(2)))
    assert set(NN_KERNELS) <= set(spills), sorted(spills)
    assert all(v == (0, 0) for v in spills.values()), {k: v for k, v in spills.items() if v != (0, 0)}


@pytest.mark.parametrize("fn", NN_KERNELS)
def test_nn_hgmma_not_serialised(compiled, fn):
    obj, _ = compiled
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", fn, obj], capture_output=True, text=True, check=True).stdout
    seq = "".join("H" if "HGMMA.64x128x16" in l else "D" for l in sass.splitlines()
                  if "HGMMA.64x128x16" in l or "WARPGROUP.DEPBAR" in l)
    assert seq.count("H") >= 2, seq
    assert not re.search(r"HD+H", seq), f"WARPGROUP.DEPBAR between HGMMAs: {seq}"
