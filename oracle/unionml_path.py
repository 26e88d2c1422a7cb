"""Oracle (test infrastructure only): the UnionML wrapper around the predictor, restated without flytekit.

``import unionml`` is impossible in this image (``flytekit`` and ``dataclasses_json`` are absent, no network), so the
dispatch logic of the reference is restated as plain functions over a small spec object.  Each function cites the
reference lines it follows; the code is written from the behaviour, not copied.

* ``default_feature_loader``   - ``unionml:unionml/dataset.py:506-520``
* ``default_feature_transformer`` - ``dataset.py:522-527``
* ``default_parser``           - ``dataset.py:489-504`` (including the 498-499 quirk: an explicit ``features`` list is
  *overridden* by "all non-target columns" whenever both are non-None)
* ``get_features``             - ``dataset.py:350-359``
* ``predict``                  - ``unionml:unionml/model.py:711-741`` dispatch,
  ``model.py:603-614`` (reader path) and ``model.py:641-650`` (features path): predictor, then callbacks whose
  exceptions are logged and swallowed
* ``serving_predict``          - ``unionml:unionml/fastapi.py:50-64`` (``get_features`` runs twice: 61 and
  ``model.py:740``)
"""
from __future__ import annotations

import json
import logging
from dataclasses import dataclass, field
from inspect import signature
from pathlib import Path
from typing import Any, Callable, List, Optional, Sequence

import pandas as pd

logger = logging.getLogger("oracle.unionml_path")


@dataclass
class PathSpec:
    """The pieces of ``Dataset`` + ``Model`` state the predict path reads."""

    reader: Optional[Callable] = None
    features: List[str] = field(default_factory=list)  # Dataset._features ([] when None was passed, dataset.py:79)
    targets: Optional[List[str]] = None
    feature_loader: Optional[Callable] = None  # None -> default
    feature_transformer: Optional[Callable] = None  # None -> default
    parser: Optional[Callable] = None  # None -> default
    parser_feature_key: int = 0
    predictor: Optional[Callable] = None
    callbacks: Sequence[Callable] = ()
    model_object: Any = None

    @property
    def data_type(self):
        # dataset.py:368-382: the reader's return annotation
        return signature(self.reader).return_annotation if self.reader is not None else None


def default_feature_loader(spec: PathSpec, features: Any) -> Any:
    if isinstance(features, Path):
        with features.open() as f:
            features = json.load(f)
    if spec.data_type is pd.DataFrame:
        data = pd.DataFrame(features)
        names = spec.features
        if not names and spec.targets is not None:
            names = [col for col in data if col not in spec.targets]
        return data[names]
    return features


def default_feature_transformer(spec: PathSpec, features: Any) -> Any:
    return features


def default_parser(spec: PathSpec, data: Any, features: Optional[List[str]], targets: Optional[List[str]]):
    if not isinstance(data, pd.DataFrame):
        return (data,)
    if features is not None and targets is not None:
        features = [col for col in data if col not in targets]
    try:
        target_data = data[targets]
    except KeyError:
        target_data = pd.DataFrame()
    return data[features], target_data


def get_features(spec: PathSpec, features: Any) -> Any:
    loaded = spec.feature_loader(features) if spec.feature_loader else default_feature_loader(spec, features)
    return spec.feature_transformer(loaded) if spec.feature_transformer else default_feature_transformer(spec, loaded)


def _run_predictor(spec: PathSpec, features: Any):
    predictions = spec.predictor(spec.model_object, features)
    for cb in spec.callbacks:
        try:
            cb(spec.model_object, features, predictions)
        except Exception as e:  # model.py:611-612 / 647-648
            logger.exception(f"Error in post-prediction callback[{cb.__name__}]: {e}")
    return predictions


def predict(spec: PathSpec, features: Any = None, **reader_kwargs):
    if features is None and not reader_kwargs:
        raise ValueError("At least one of features or **reader_kwargs needs to be provided")
    if spec.model_object is None:
        raise RuntimeError(
            "ModelArtifact not found. You must train a model first with the `train` method before generating "
            "predictions."
        )
    if features is None:
        data = spec.reader(**reader_kwargs)
        if spec.parser:
            parsed = spec.parser(data, features=spec.features, targets=spec.targets)
        else:
            parsed = default_parser(spec, data, spec.features, spec.targets)
        feats = parsed[spec.parser_feature_key]
        feats = spec.feature_transformer(feats) if spec.feature_transformer else feats
        return _run_predictor(spec, feats)
    return _run_predictor(spec, get_features(spec, features))


def serving_predict(spec: PathSpec, inputs: Optional[dict] = None, features: Optional[list] = None):
    """Body of ``POST /predict``; raises ``LookupError`` where the reference raises ``HTTPException(500)``."""
    if inputs is None and features is None:
        raise LookupError("inputs or features must be supplied.")
    workflow_inputs: dict = {}
    if spec.data_type is not None:
        features = get_features(spec, features)
    workflow_inputs.update(inputs if inputs else {"features": features})
    return predict(spec, **workflow_inputs)
