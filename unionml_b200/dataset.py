"""``Dataset``: the data side of the decorator protocol, for the predict (and local train) slice.

Mirrors the public surface of ``unionml:unionml/dataset.py`` that the hot path touches - ``reader``,
``loader``, ``splitter``, ``parser``, ``feature_loader``, ``feature_transformer``, ``get_data``, ``get_features`` -
with the same defaults and the same quirks, but without flytekit: functions are plain closures called in-process
(the reference wraps each in a flytekit task and round-trips every DataFrame through a StructuredDataset).

Out of scope here (SURVEY.md section 2): ``from_sqlite_task`` / ``from_sqlalchemy_task`` and the kwargs dataclasses
that exist only to give Flyte workflows typed inputs.
"""

import json
from functools import partial
from inspect import Parameter, signature
from pathlib import Path
from typing import Any, Callable, Dict, List, Optional, Tuple, Type, get_args

import pandas as pd

from unionml_b200 import type_guards


class Dataset:
    def __init__(
        self,
        name: str = "dataset",
        *,
        features: Optional[List[str]] = None,
        targets: Optional[List[str]] = None,
        test_size: float = 0.2,
        shuffle: bool = True,
        random_state: int = 12345,
    ):
        # same defaults as unionml:unionml/dataset.py:44-53
        self.name = name
        self._features: List[str] = [] if features is None else features
        self._targets = targets
        self._test_size = test_size
        self._shuffle = shuffle
        self._random_state = random_state

        self._reader: Optional[Callable] = None
        self._loader: Callable = self._default_loader
        self._splitter: Callable = self._default_splitter
        self._parser: Callable = self._default_parser
        self._parser_feature_key = 0
        self._feature_loader: Callable = self._default_feature_loader
        self._feature_transformer: Callable = self._default_feature_transformer
        self._reader_task_kwargs: Dict[str, Any] = {}

    # ---------------------------------------------------------------------------------------------------------
    # decorators (ref. dataset.py:103-212)
    # ---------------------------------------------------------------------------------------------------------
    def reader(self, fn=None, **reader_task_kwargs):
        if fn is None:
            return partial(self.reader, **reader_task_kwargs)
        type_guards.guard_reader(fn)
        self._reader = fn
        self._reader_task_kwargs = dict(reader_task_kwargs)  # resource requests etc.: accepted, unused locally
        return fn

    def loader(self, fn):
        type_guards.guard_loader(fn, self.dataset_datatype["data"])
        self._loader = fn
        return fn

    def splitter(self, fn):
        type_guards.guard_splitter(fn, self.dataset_datatype["data"], self.dataset_datatype_source)
        self._splitter = fn
        return fn

    def parser(self, fn, feature_key: int = 0):
        type_guards.guard_parser(fn, self.dataset_datatype["data"], self.dataset_datatype_source)
        self._parser = fn
        self._parser_feature_key = feature_key
        return fn

    def feature_loader(self, fn):
        type_guards.guard_feature_loader(fn, Any)
        self._feature_loader = fn
        return fn

    def feature_transformer(self, fn):
        type_guards.guard_feature_transformer(fn, signature(self._feature_loader).return_annotation)
        self._feature_transformer = fn
        return fn

    # ---------------------------------------------------------------------------------------------------------
    # kwargs forwarded to splitter / parser (ref. dataset.py:214-229)
    # ---------------------------------------------------------------------------------------------------------
    @property
    def splitter_kwargs(self) -> Dict[str, Any]:
        return {"test_size": self._test_size, "shuffle": self._shuffle, "random_state": self._random_state}

    @property
    def parser_kwargs(self) -> Dict[str, Any]:
        return {"features": self._features, "targets": self._targets}

    # ---------------------------------------------------------------------------------------------------------
    # types (ref. dataset.py:361-424)
    # ---------------------------------------------------------------------------------------------------------
    @property
    def dataset_datatype(self) -> Dict[str, Type]:
        if self._loader != self._default_loader:
            return {"data": signature(self._loader).return_annotation}
        if self._reader is not None:
            return {"data": signature(self._reader).return_annotation}
        raise ValueError(
            "dataset_datatype is not defined. Please define a @dataset.reader function with an output annotation."
        )

    @property
    def dataset_datatype_source(self) -> str:
        return "loader" if self._loader != self._default_loader else "reader"

    @property
    def reader_input_types(self) -> Optional[List[Parameter]]:
        return None if self._reader is None else [*signature(self._reader).parameters.values()]

    @property
    def parser_return_types(self) -> Tuple[Any, ...]:
        return get_args(signature(self._parser).return_annotation)

    @property
    def feature_type(self) -> Type:
        dataset_type = (
            self.dataset_datatype["data"]
            if self._parser == self._default_parser
            else self.parser_return_types[self._parser_feature_key]
        )
        if self._feature_loader == self._default_feature_loader:
            return dataset_type
        produced = (
            signature(self._feature_loader).return_annotation
            if self._feature_transformer == self._default_feature_transformer
            else signature(self._feature_transformer).return_annotation
        )
        if dataset_type != produced:
            # the reference returns FeatureTypeUnion[dataset_type, produced]; for guard purposes a typing.Union
            # has the same "appears among the arguments" behaviour
            from typing import Union

            return Union[dataset_type, produced]  # type: ignore[return-value]
        return dataset_type

    # ---------------------------------------------------------------------------------------------------------
    # execution (ref. dataset.py:302-359)
    # ---------------------------------------------------------------------------------------------------------
    def read(self, **reader_kwargs):
        """What the reference's ``dataset_task`` does (ref. 282-300): call the registered reader."""
        if self._reader is None:
            raise ValueError("No @dataset.reader registered.")
        return self._reader(**reader_kwargs)

    def get_data(
        self,
        raw_data,
        loader_kwargs: Optional[Dict[str, Any]] = None,
        splitter_kwargs: Optional[Dict[str, Any]] = None,
        parser_kwargs: Optional[Dict[str, Any]] = None,
    ) -> Dict[str, Any]:
        merged = lambda base, new: base if new is None else {**base, **new}  # noqa: E731
        data = self._loader(raw_data, **merged({}, loader_kwargs))
        splits = self._splitter(data, **merged(self.splitter_kwargs, splitter_kwargs))
        pk = merged(self.parser_kwargs, parser_kwargs)
        out = {}
        for key, split in zip(("train", "test"), splits):
            parsed = [*self._parser(split, **pk)]
            parsed[self._parser_feature_key] = self._feature_transformer(parsed[self._parser_feature_key])
            out[key] = parsed
        return out

    def get_features(self, features):
        """feature_loader -> feature_transformer (ref. dataset.py:350-359)."""
        return self._feature_transformer(self._feature_loader(features))

    # ---------------------------------------------------------------------------------------------------------
    # defaults (behaviour of ref. dataset.py:472-527; pandas frames are the only structure handled natively)
    # ---------------------------------------------------------------------------------------------------------
    def _frames_are_native(self) -> bool:
        return self.dataset_datatype["data"] is pd.DataFrame

    def _default_loader(self, data: Any) -> Any:
        return pd.DataFrame(data) if self._frames_are_native() else data

    def _default_splitter(self, data: Any, test_size: float, shuffle: bool, random_state: int) -> Tuple[Any, ...]:
        if isinstance(data, pd.DataFrame):
            from sklearn.model_selection import train_test_split

            train, test = train_test_split(data, test_size=test_size, random_state=random_state, shuffle=shuffle)
            return train, test
        return (data,)

    def _default_parser(self, data: Any, features: Optional[List[str]], targets: Optional[List[str]]) -> Tuple[Any, ...]:
        if not isinstance(data, pd.DataFrame):
            return (data,)
        # Quirk kept on purpose (ref. 498-499): whenever a target list exists, an explicit feature list is replaced by
        # "every column that is not a target".
        feature_cols = features
        if features is not None and targets is not None:
            feature_cols = [c for c in data.columns if c not in targets]
        target_frame = data[targets] if _has_columns(data, targets) else pd.DataFrame()
        return data[feature_cols], target_frame

    def _default_feature_loader(self, features: Any) -> Any:
        raw = json.loads(features.read_text()) if isinstance(features, Path) else features
        if not self._frames_are_native():
            return raw
        frame = pd.DataFrame(raw)
        wanted = self._features
        if not wanted and self._targets is not None:
            wanted = [c for c in frame.columns if c not in self._targets]
        if wanted is not None and len(wanted) == frame.shape[1] and list(wanted) == list(frame.columns):
            # the selection is the identity (same columns, same order): hand the frame through instead of letting
            # `frame[wanted]` copy every block - a 10M x 64 float64 frame is 5 GB (SURVEY.md 8a row a2 "where time goes")
            return frame
        return frame[wanted]

    def _default_feature_transformer(self, features: Any) -> Any:
        return features  # identity unless @dataset.feature_transformer is registered


def _has_columns(frame: pd.DataFrame, names: Optional[List[str]]) -> bool:
    """``frame[names]`` would succeed (the reference catches the KeyError instead, ref. 500-503)."""
    try:
        frame[names]
        return True
    except KeyError:
        return False
