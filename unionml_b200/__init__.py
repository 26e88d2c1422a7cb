"""unionml_b200: an H100-native engine for UnionML's ``Model.predict`` / ``@model.predictor`` hot path.

Keeps the reference's decorator surface for the predict slice (``Dataset``, ``Model``, ``@model.predictor``, callbacks,
``serving_app``) and runs the canonical ``LogisticRegression`` predictor as hand-written sm_90a CUDA behind a C ABI
(``include/uml_b200.h``).  Importing this package never touches CUDA; the device is bound on first predict.
"""
from unionml_b200.dataset import Dataset  # noqa: F401
from unionml_b200.model import Model, ModelArtifact  # noqa: F401

__all__ = ["Dataset", "Model", "ModelArtifact"]
