"""The study's four case studies for PyTorch models (case_study.py, case_study_{mnist,fashion_mnist,cifar10,imdb}.py):
their networks, training recipes, layer choices and datasets, and a runner for the reference's phases."""
from __future__ import annotations

from .base import CaseStudy, load_state, model_path
from .cifar10 import Cifar10CaseStudy
from .fmnist import FashionMnistCaseStudy
from .imdb import ImdbCaseStudy
from .mnist import MnistCaseStudy

CASE_STUDIES = {c.name: c for c in (MnistCaseStudy, FashionMnistCaseStudy, Cifar10CaseStudy, ImdbCaseStudy)}


def load_model(output_folder: str, name: str, model_id: int, device="cuda"):
    """The network of case study `name` with the weights `CaseStudy.train` saved for `model_id`, in eval mode."""
    return load_state(CASE_STUDIES[name].network(), model_path(output_folder, name, model_id), device)
