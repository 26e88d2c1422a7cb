"""``Model``: the model side of the decorator protocol with a local, in-process executor.

Mirrors the surface of ``unionml:unionml/model.py`` that the predict hot path (and the local ``train`` of the
README digits app) touches: ``init / trainer / predictor / evaluator / saver / loader`` decorators, prediction
callbacks, ``train``, ``predict``, ``save``, ``load``, ``load_from_env``, ``serve``, ``resolve_model_artifact``.

What is different by design: ``Model.predict`` does not build a flytekit ``Workflow`` per call
(ref. ``model.py:497-510, 736-741``) and does not push the feature frame through Flyte literals; it calls the
registered closures directly, in the order the reference's tasks do (ref. ``model.py:603-614`` reader path,
``641-650`` features path).  The drop-in boundary is the same single call: ``self._predictor(model_object, features)``.

Out of scope (SURVEY.md section 2): remote deploy/train/predict, schedules, Flyte task/workflow objects.
"""

import inspect
import os
from dataclasses import asdict, is_dataclass, make_dataclass
from functools import partial
from inspect import Parameter, signature
from typing import IO, Any, Callable, Dict, List, NamedTuple, Optional, Tuple, Type, Union

import pandas as pd

from unionml_b200 import type_guards
from unionml_b200._logging import logger
from unionml_b200.dataset import Dataset


class ModelArtifact(NamedTuple):
    """Model object plus optional hyperparameters and metrics (ref. ``model.py:46-56``)."""

    model_object: Any
    hyperparameters: Optional[Union[dict, Any]] = None
    metrics: Optional[Dict[str, float]] = None


def _is_pytorch_model(model_type) -> bool:
    try:
        import torch.nn as nn

        return inspect.isclass(model_type) and issubclass(model_type, nn.Module)
    except Exception:  # torch absent
        return False


class Model:
    def __init__(
        self,
        name: str = "model",
        init: Union[Type, Callable, None] = None,
        *,
        dataset: Dataset,
        hyperparameter_config: Optional[Dict[str, Type]] = None,
    ):
        self.name = name
        self._init_callable = init
        self._hyperparameter_config = hyperparameter_config
        self._dataset = dataset
        self._artifact: Optional[ModelArtifact] = None

        self._init: Callable = self._default_init
        self._saver: Callable = self._default_saver
        self._loader: Callable = self._default_loader
        self._trainer: Optional[Callable] = None
        self._predictor: Optional[Callable] = None
        self._evaluator: Optional[Callable] = None
        self._predict_callbacks: Tuple[Callable, ...] = ()
        self._train_task_kwargs: Dict[str, Any] = {}
        self._predict_task_kwargs: Dict[str, Any] = {}
        self._hyperparameter_type: Optional[Type] = None

        if self._dataset.name is None:
            self._dataset.name = f"{self.name}.dataset"

    # ---------------------------------------------------------------------------------------------------------
    # properties
    # ---------------------------------------------------------------------------------------------------------
    @property
    def artifact(self) -> Optional[ModelArtifact]:
        return self._artifact

    @artifact.setter
    def artifact(self, new_value: ModelArtifact):
        self._artifact = new_value

    @property
    def dataset(self) -> Dataset:
        return self._dataset

    @property
    def predict_callbacks(self) -> Tuple[Callable, ...]:
        return self._predict_callbacks

    @predict_callbacks.setter
    def predict_callbacks(self, value):
        self._predict_callbacks = tuple(value)

    @property
    def model_type(self) -> Type:
        # ref. model.py:1420-1423
        init = self._init_callable if self._init == self._default_init else self._init or self._init_callable
        if inspect.isclass(init):
            return init
        return signature(init).return_annotation if init is not None else init

    @property
    def prediction_type(self) -> Type:
        return signature(self._predictor).return_annotation

    @property
    def hyperparameter_type(self) -> Type:
        """A dataclass of the hyperparameters (ref. ``model.py:181-212``); used by ``save``/``load`` round trips."""
        if self._hyperparameter_type is not None:
            return self._hyperparameter_type
        fields: List[Any] = []
        if self._hyperparameter_config is not None:
            fields = [(k, v) for k, v in self._hyperparameter_config.items()]
        elif self._init_callable is not None:
            for p in signature(self._init_callable).parameters.values():
                if p.kind in (Parameter.VAR_KEYWORD, Parameter.VAR_POSITIONAL) or p.name == "self":
                    continue
                ann = Any if p.annotation is Parameter.empty else p.annotation
                if p.default is Parameter.empty:
                    fields.append((p.name, ann))
                else:
                    from dataclasses import field

                    default = p.default
                    if isinstance(default, (list, dict, set)):
                        fields.append((p.name, ann, field(default_factory=lambda d=default: d)))
                    else:
                        fields.append((p.name, ann, field(default=default)))
            fields.sort(key=lambda f: len(f) == 3)  # required fields first
        self._hyperparameter_type = make_dataclass("Hyperparameters", fields)
        return self._hyperparameter_type

    # ---------------------------------------------------------------------------------------------------------
    # decorators (ref. model.py:256-414)
    # ---------------------------------------------------------------------------------------------------------
    def init(self, fn):
        self._init = fn
        return self._init

    def _expected_data_types(self):
        if self._dataset._parser == self._dataset._default_parser:
            dt = self._dataset.dataset_datatype["data"]
            return (dt, dt) if dt is pd.DataFrame else (dt,)
        return self._dataset.parser_return_types

    def trainer(self, fn: Optional[Callable] = None, **train_task_kwargs):
        if fn is None:
            return partial(self.trainer, **train_task_kwargs)
        type_guards.guard_trainer(fn, self.model_type, self._expected_data_types())
        self._trainer = fn
        self._train_task_kwargs = dict(train_task_kwargs)
        if not hasattr(fn, "__unionml_model__"):
            fn.__unionml_model__ = self
        return fn

    def predictor(self, fn=None, callbacks: Optional[List[Callable]] = None, **predict_task_kwargs):
        """Register the function behind the drop-in boundary (ref. ``model.py:319-367``)."""
        if fn is None:
            return partial(self.predictor, callbacks=callbacks, **predict_task_kwargs)
        model_t, feature_t = self.model_type, self._dataset.feature_type
        type_guards.guard_predictor(fn, model_t, feature_t)
        self._predictor = fn
        self._predict_task_kwargs = dict(predict_task_kwargs)
        # callbacks are checked against the predictor's return annotation, so they are validated after it
        checked = []
        for cb in callbacks or ():
            if not callable(cb):
                raise ValueError("Callback must be a callable function.")
            type_guards.guard_prediction_callback(
                callback=cb, predictor=fn, expected_model_type=model_t, expected_data_type=feature_t
            )
            checked.append(cb)
        if callbacks is not None:
            self.predict_callbacks = checked
        try:
            if not hasattr(fn, "__unionml_model__"):
                fn.__unionml_model__ = self  # lets decorators stacked on top find the model
        except AttributeError:  # builtins / bound methods do not take attributes
            pass
        return fn

    def evaluator(self, fn):
        type_guards.guard_evaluator(fn, self.model_type, self._expected_data_types())
        self._evaluator = fn
        return fn

    def saver(self, fn):
        self._saver = fn
        return fn

    def loader(self, fn):
        self._loader = fn
        return fn

    @property
    def trainer_params(self) -> Dict[str, Parameter]:
        return {
            n: p for n, p in signature(self._trainer).parameters.items() if p.kind == Parameter.KEYWORD_ONLY
        }

    # ---------------------------------------------------------------------------------------------------------
    # local execution
    # ---------------------------------------------------------------------------------------------------------
    def train(
        self,
        hyperparameters: Optional[Dict[str, Any]] = None,
        loader_kwargs: Optional[Dict[str, Any]] = None,
        splitter_kwargs: Optional[Dict[str, Any]] = None,
        parser_kwargs: Optional[Dict[str, Any]] = None,
        trainer_kwargs: Optional[Dict[str, Any]] = None,
        **reader_kwargs,
    ) -> Tuple[Any, Any]:
        """reader -> loader -> splitter -> parser -> trainer -> evaluator per split (ref. ``model.py:560-575, 655-709``)."""
        trainer_kwargs = {} if trainer_kwargs is None else trainer_kwargs
        hyperparameters = {} if hyperparameters is None else hyperparameters
        hp_dict = asdict(hyperparameters) if is_dataclass(hyperparameters) else dict(hyperparameters)
        raw = self._dataset.read(**reader_kwargs)
        data = self._dataset.get_data(raw, loader_kwargs, splitter_kwargs, parser_kwargs)
        model_object = self._trainer(self._init(hyperparameters=hp_dict), *data["train"], **trainer_kwargs)
        metrics = {split: self._evaluator(model_object, *data[split]) for split in data}
        self.artifact = ModelArtifact(model_object, hp_dict, metrics)
        return model_object, metrics

    def _run_predictor(self, model_object, features):
        predictions = self._predictor(model_object, features)  # <- the drop-in boundary (ref. model.py:606, 642)
        for callback in self.predict_callbacks:
            try:
                callback(model_object, features, predictions)
            except Exception as e:  # logged and swallowed, like ref. model.py:608-612
                logger.exception(f"Error in post-prediction callback[{callback.__name__}]: {e}")
        return predictions

    def predict(self, features: Any = None, **reader_kwargs):
        """Generate predictions locally (ref. ``model.py:711-741``)."""
        if features is None and not reader_kwargs:
            raise ValueError("At least one of features or **reader_kwargs needs to be provided")
        if self.artifact is None:
            raise RuntimeError(
                "ModelArtifact not found. You must train a model first with the `train` method before generating "
                "predictions."
            )
        if features is None:
            ds = self._dataset
            parsed = ds._parser(ds.read(**reader_kwargs), **ds.parser_kwargs)
            feats = ds._feature_transformer(parsed[ds._parser_feature_key])
        else:
            feats = self._dataset.get_features(features)
        return self._run_predictor(self.artifact.model_object, feats)

    # ---------------------------------------------------------------------------------------------------------
    # persistence (ref. model.py:743-769, 1432-1519)
    # ---------------------------------------------------------------------------------------------------------
    def save(self, file: Union[str, os.PathLike, IO], *args, **kwargs):
        if self.artifact is None:
            raise AttributeError("`artifact` property is None. Call the `train` method to train a model first")
        return self._saver(self.artifact.model_object, self.artifact.hyperparameters, file, *args, **kwargs)

    def load(self, file: Union[str, os.PathLike, IO], *args, **kwargs):
        self.artifact = ModelArtifact(self._loader(file, *args, **kwargs))
        return self.artifact.model_object

    def load_from_env(self, env_var: str = "UNIONML_MODEL_PATH", *args, **kwargs):
        model_path = os.getenv(env_var)
        if model_path is None:
            raise ValueError(f"env_var for model path {env_var} doesn't exist.")
        return self.load(model_path)

    def serve(self, app, remote: bool = False, app_version: Optional[str] = None, model_version: str = "latest"):
        """Attach ``/predict`` and ``/health`` to a FastAPI app (ref. ``model.py:771-784``)."""
        from unionml_b200.fastapi import serving_app

        serving_app(self, app, remote=remote, app_version=app_version, model_version=model_version)

    def resolve_model_artifact(
        self,
        model_object: Optional[Any] = None,
        model_version: Optional[str] = None,
        app_version: Optional[str] = None,
        model_file: Optional[Union[str, os.PathLike]] = None,
        loader_kwargs: Optional[dict] = None,
    ) -> ModelArtifact:
        sources = {"model_object": model_object, "model_version": model_version, "model_file": model_file}
        given = [k for k, v in sources.items() if v is not None]
        if len(given) > 1:
            raise ValueError("You can specify only one of 'model_object', 'model_version', or 'model_file' arguments.")
        if not given:
            if self.artifact is None:
                raise ValueError(
                    "Model object not found. Make sure to specify at least one of model_version, model_file, or "
                    "model_object. Alternatively, train a model locally with the .train(...) method so the "
                    "model.artifact property contains a model object."
                )
            return self.artifact
        if given[0] == "model_object":
            return ModelArtifact(model_object)
        if given[0] == "model_file":
            return ModelArtifact(self.load(model_file, **(loader_kwargs or {})))
        raise NotImplementedError("Fetching artifacts from a Flyte cluster is out of scope for unionml_b200.")

    def _default_init(self, hyperparameters: dict) -> Any:
        if self._init_callable is None:
            raise ValueError(
                "When using the _default_init method, you must specify the init argument to the Model constructor."
            )
        return self._init_callable(**hyperparameters)

    def _default_saver(self, model_obj: Any, hyperparameters, file, *args, **kwargs) -> Any:
        import sklearn.base

        if hyperparameters is not None and is_dataclass(hyperparameters):
            hyperparameters = asdict(hyperparameters)
        if isinstance(model_obj, sklearn.base.BaseEstimator):
            import joblib

            return joblib.dump({"model_obj": model_obj, "hyperparameters": hyperparameters}, file, *args, **kwargs)
        if _is_pytorch_model(self.model_type):
            import torch

            torch.save({"model_obj": model_obj.state_dict(), "hyperparameters": hyperparameters}, file, *args, **kwargs)
            return file
        raise NotImplementedError(
            f"Default saver not defined for type {type(model_obj)}. Use the Model.saver decorator to define one."
        )

    def _default_loader(self, file, *args, **kwargs) -> Any:
        import sklearn.base

        model_type = self.model_type
        if inspect.isclass(model_type) and issubclass(model_type, sklearn.base.BaseEstimator):
            import joblib

            return joblib.load(file, *args, **kwargs)["model_obj"]
        if _is_pytorch_model(model_type):
            import torch

            blob = torch.load(file, *args, **kwargs)
            hp = blob["hyperparameters"]
            model = self._init(hp) if self._init_callable is not None else model_type(**hp)
            model.load_state_dict(blob["model_obj"])
            return model
        raise NotImplementedError(
            f"Default loader not defined for type {model_type}. Use the Model.loader decorator to define one."
        )
