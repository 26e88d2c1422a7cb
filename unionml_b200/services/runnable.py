"""The runner entry point of the reference's BentoML binding, without BentoML.

``unionml:unionml/services/bentoml.py:190-213`` defines ``UnionMLRunnable.predict`` as::

    features = self.model.dataset.get_features(features)
    return self.model.predict(features=features)

(``get_features`` runs twice - there and inside ``Model.predict``.)  BentoML itself (service packaging, IO
descriptors, ``bentoml serve``) is a third-party server that is not installed in this image and is out of scope;
what is kept is the call site, so a BentoML ``Runnable`` can subclass/wrap :class:`PredictRunnable` unchanged.
"""

from typing import Any, Optional, Tuple

from unionml_b200.model import Model


class PredictRunnable:
    SUPPORTED_RESOURCES: Tuple[str, ...] = ("cpu", "nvidia.com/gpu")  # ref. bentoml.py:202
    SUPPORTS_CPU_MULTI_THREADING = False  # ref. bentoml.py:203

    def __init__(self, model: Model):
        self.model = model

    def predict(self, features: Any) -> Any:
        features = self.model.dataset.get_features(features)
        return self.model.predict(features=features)


def create_runnable(
    supported_resources: Optional[Tuple[str, ...]] = None,
    supports_cpu_multi_threading: bool = False,
):
    """Class factory with the reference's knobs (ref. ``bentoml.py:190-213``)."""

    class _Runnable(PredictRunnable):
        SUPPORTED_RESOURCES = supported_resources or PredictRunnable.SUPPORTED_RESOURCES
        SUPPORTS_CPU_MULTI_THREADING = supports_cpu_multi_threading

    return _Runnable
