"""Registration-time signature checks for the decorator protocol.

Same contract as the reference's guards (``unionml:unionml/type_guards.py``): a mismatch raises ``TypeError``
when the function is *registered*, never at predict time.  The rules that matter to the predict path:

* ``guard_predictor`` (ref. 151-169): first parameter = model type, exactly one positional ``features`` parameter
  compatible with the dataset's feature type, and a return annotation is mandatory.
* ``guard_prediction_callback`` (ref. 172-232): ``(model_object, features, predictions) -> None``.
* ``guard_feature_loader`` / ``guard_feature_transformer`` (ref. 235-254): exactly one parameter.
* ``guard_reader`` (ref. 81-88): a return annotation is mandatory (it defines the dataset datatype).

"Compatible" (ref. 28-41): equal, either side ``Any``, or one type appears among the other's ``typing`` arguments.
"""
from __future__ import annotations

from inspect import Parameter, Signature, signature
from typing import Any, Callable, Iterable, List, Optional, Type, get_args, get_origin

_EMPTY = Signature.empty
_POSITIONAL = (Parameter.POSITIONAL_OR_KEYWORD, Parameter.POSITIONAL_ONLY)


def compatible(actual: Any, expected: Any) -> bool:
    if actual is Any or expected is Any:
        return True
    return actual == expected or expected in get_args(actual) or actual in get_args(expected)


def _require_compatible(fn_name: str, actual: Any, expected: Any) -> None:
    if not compatible(actual, expected):
        raise TypeError(
            f"The type of the first argument of the '{fn_name}' function must be compatible with the expected output "
            f"type: {expected}. Found {actual}"
        )


def _split_params(fn: Callable):
    params = list(signature(fn).parameters.values())
    head = params[0].annotation if params else _EMPTY
    data = [p.annotation for p in params[1:] if p.kind in _POSITIONAL]
    return head, data


def guard_reader(reader: Callable) -> None:
    if signature(reader).return_annotation is _EMPTY:
        raise TypeError(
            "The dataset.reader function return annotation cannot be empty. You need to specify a return type."
        )


def guard_loader(loader: Callable, expected_data_type: Type) -> None:
    head, _ = _split_params(loader)
    _require_compatible("loader", head, expected_data_type)


def _is_sequence_type(tp: Any) -> bool:
    return get_origin(tp) in {tuple, list} or getattr(tp, "__bases__", None) == (tuple,)


def guard_splitter(splitter: Callable, expected_data_type: Type, expected_type_source: str) -> None:
    sig = signature(splitter)
    head, _ = _split_params(splitter)
    _require_compatible("splitter", head, expected_data_type)
    out = sig.return_annotation
    if not _is_sequence_type(out):
        raise TypeError(
            f"The output of 'splitter' must be a List, Tuple, or NamedTuple type containing data splits. Found {out}"
        )
    for sub in get_args(out):
        if sub != expected_data_type:
            raise TypeError(
                f"The type arguments to the output generic type of 'splitter' the function must match the "
                f"'{expected_type_source}' output type: {expected_data_type}. Found {out}"
            )
    _require_kwargs("splitter", sig, {"test_size": float, "shuffle": bool, "random_state": int})


def guard_parser(parser: Callable, expected_data_type: Type, expected_type_source: str) -> None:
    sig = signature(parser)
    head, _ = _split_params(parser)
    _require_compatible("parser", head, expected_data_type)
    if not _is_sequence_type(sig.return_annotation):
        raise TypeError(
            "The output of 'parser' must be a List, Tuple, or NamedTuple type containing data splits. "
            f"Found {sig.return_annotation}"
        )
    _require_kwargs("parser", sig, {"features": Optional[List[str]], "targets": List[str]})


def _require_kwargs(fn_name: str, sig: Signature, kwtypes: dict) -> None:
    for pos, (name, tp) in enumerate(kwtypes.items(), start=1):
        param = sig.parameters.get(name)
        if param is None:
            raise TypeError(
                f"The '{fn_name}' function is expected to accept an argument '{name}' of type {tp} at the {pos}th "
                f"position. Found a function with the following signature: {sig.parameters}"
            )
        if param.annotation != tp:
            raise TypeError(f"The argument '{name}' expected to be of type {tp}, found {param.annotation}")


def _guard_model_and_data(fn_name: str, fn: Callable, model_type: Type, data_types: Iterable[Type]) -> None:
    head, data = _split_params(fn)
    data_types = tuple(data_types)
    _require_compatible(fn_name, head, model_type)
    if len(data) != len(data_types):
        raise TypeError(f"Length of positional data arguments are expected to match {data_types}. Found {data}.")
    for actual, expected in zip(data, data_types):
        _require_compatible(fn_name, actual, expected)


def guard_trainer(trainer: Callable, expected_model_type: Type, expected_data_types: Iterable[Type]) -> None:
    _guard_model_and_data("trainer", trainer, expected_model_type, expected_data_types)
    _require_compatible("trainer", signature(trainer).return_annotation, expected_model_type)


def guard_evaluator(evaluator: Callable, expected_model_type: Type, expected_data_types: Iterable[Type]) -> None:
    _guard_model_and_data("evaluator", evaluator, expected_model_type, expected_data_types)


def guard_predictor(predictor: Callable, expected_model_type: Type, expected_data_type: Type) -> None:
    head, data = _split_params(predictor)
    if len(data) != 1:
        raise TypeError(f"The 'predictor' function must take a single 'features' argument, found {data}")
    _require_compatible("predictor", head, expected_model_type)
    _require_compatible("predictor", data[0], expected_data_type)
    if signature(predictor).return_annotation is _EMPTY:
        raise TypeError("The 'predictor' function needs a return type annotation.")


def guard_prediction_callback(
    callback: Callable, predictor: Callable, expected_model_type: Type, expected_data_type: Type
) -> None:
    name = getattr(callback, "__name__", repr(callback))
    prediction_type = signature(predictor).return_annotation
    if prediction_type is _EMPTY:
        raise TypeError("The 'predictor' function needs a return type annotation.")
    ret = signature(callback).return_annotation
    if ret is not _EMPTY and ret is not None:
        raise TypeError(f"The 'callback[{name}]' function must have None as it's return annotation.")
    head, data = _split_params(callback)
    if len(data) != 2:
        raise TypeError(
            f"Callback functions (callback[{name}]) must take both 'features' and 'prediction' arguments, found {data}"
        )
    for position, actual, expected in (
        ("first", head, expected_model_type),
        ("second", data[0], expected_data_type),
        ("third", data[1], prediction_type),
    ):
        if not compatible(actual, expected):
            raise TypeError(
                f"The type of the {position} argument of the callback[{name}] function must be compatible with the "
                f"expected output type: {expected}. Found {actual}"
            )


def _guard_single_arg(fn_name: str, fn: Callable, expected_data_type: Type, what: str) -> None:
    params = list(signature(fn).parameters.values())
    if len(params) != 1:
        raise TypeError(f"The '{fn_name}' must take a single argument representing {what}.")
    _require_compatible(fn_name, params[0].annotation, expected_data_type)


def guard_feature_loader(feature_loader: Callable, expected_data_type: Type) -> None:
    _guard_single_arg("feature_loader", feature_loader, expected_data_type, "raw features or a reference to raw features")


def guard_feature_transformer(feature_transformer: Callable, expected_data_type: Type) -> None:
    _guard_single_arg("feature_transformer", feature_transformer, expected_data_type, "the loaded features")
