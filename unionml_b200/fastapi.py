"""FastAPI binding of the device predict path: ``POST /predict``, ``GET /health``, ``GET /``.

Behaviour follows ``unionml:unionml/fastapi.py:15-70``:

* at startup the model object is loaded from ``UNIONML_MODEL_PATH`` unless the ``Model`` already carries an artifact
  (ref. 22-34).  The CUDA engine is *not* touched here: it is bound lazily by the first predict inside the worker
  process (``unionml serve --workers N`` forks, ``cli.py:289``);
* ``/predict`` accepts ``{"features": [...]}`` (records) or ``{"inputs": {...reader kwargs}}``; with neither it answers
  HTTP 500 (ref. 55-56).  Features pass through ``Dataset.get_features`` here *and again* inside ``Model.predict``
  (ref. 61 and ``model.py:740``) - kept, the default loader is idempotent;
* ``/health`` answers 500 until an artifact exists (ref. 66-70).

Artifacts fetched from a Flyte cluster (``remote=True``) are out of scope.
"""
import os
from http import HTTPStatus
from typing import Any, Dict, List, Optional

from fastapi import Body, FastAPI, HTTPException
from fastapi.responses import HTMLResponse

from unionml_b200.model import Model, ModelArtifact

_INDEX_PAGE = (
    "<html><head><title>unionml</title></head>"
    "<body><h1>unionml</h1><p>H100 batch-prediction engine behind the UnionML predictor API</p></body></html>"
)
_NO_MODEL_PATH = (
    "Model artifact path not specified. Make sure to specify the unionml serve --model-path in "
    "the option when starting the unionml prediction service in local mode."
)


class _PredictionService:
    """The three route handlers, bound to one ``Model``."""

    def __init__(self, model: Model):
        self.model = model

    def load_artifact(self) -> None:
        if self.model.artifact is not None:
            return
        path = os.getenv("UNIONML_MODEL_PATH")
        if path is None:
            raise ValueError(_NO_MODEL_PATH)
        self.model.artifact = ModelArtifact(self.model.load(path))

    def index(self) -> str:
        return _INDEX_PAGE

    async def predict(
        self,
        inputs: Optional[Dict[str, Any]] = Body(None),
        features: Optional[List[Any]] = Body(None),
    ):
        if features is None and inputs is None:
            raise HTTPException(status_code=500, detail="inputs or features must be supplied.")
        dataset = self.model.dataset
        if dataset.dataset_datatype is not None:  # first get_features; Model.predict applies it a second time
            features = dataset.get_features(features)
        call_kwargs = dict(inputs) if inputs else {"features": features}
        return self.model.predict(**call_kwargs)

    async def health(self):
        if self.model.artifact is None:
            raise HTTPException(status_code=500, detail="Model artifact not found.")
        ok = HTTPStatus.OK
        return {"message": ok.phrase, "status": ok}


def serving_app(
    model: Model,
    app: FastAPI,
    remote: bool = False,
    app_version: Optional[str] = None,
    model_version: str = "latest",
):
    """Attach the prediction routes of ``model`` to ``app`` (what ``Model.serve`` calls)."""
    if remote:
        raise NotImplementedError("remote=True (Flyte-backed artifacts) is out of scope for unionml_b200")
    service = _PredictionService(model)
    app.router.on_startup.append(service.load_artifact)
    app.add_api_route("/", service.index, methods=["GET"], response_class=HTMLResponse)
    app.add_api_route("/predict", service.predict, methods=["POST"])
    app.add_api_route("/health", service.health, methods=["GET"])
    return app
