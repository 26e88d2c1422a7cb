"""cfg 4 of BASELINE.json: FastAPI /predict online serving, batch = 32, p50 / p99 latency on 1 x H100 - with the
reference-shaped CPU predictor served through the SAME app beside it (one JSON line; not part of the driver contract).

    python tools/bench_online.py [--requests 1000] [--app linear|mlp]

Both apps are `unionml_b200.Model.serve(FastAPI())` (mirror of unionml:unionml/fastapi.py:15-70) driven by the
in-process ASGI TestClient with 1 000 POSTs of digits.frame[features].sample(32, random_state=i) records (SURVEY.md 8d).
--app linear (the scikit-learn digits app):
  * device : @model.predictor = unionml_b200.predictors.linear_argmax  (small-batch float64 kernel, CUDA graph replay)
  * cpu    : @model.predictor = [float(x) for x in estimator.predict(features)]  (unionml:README.md:87-92)
--app mlp (the torch quickstart app, PytorchModel(64, 32, 10) with torch.manual_seed(0): tests/golden/mlp_64_32_10.npz):
  * device : @model.predictor = unionml_b200.predictors.mlp_argmax  (the same online route with mlp_small_kernel)
  * torch  : @model.predictor = [float(x) for x in module(torch.from_numpy(features.values).float()).argmax(1)]
and the predictor call alone is timed for both (what the device path changes inside a request).  The mlp run also
times the engine call on 65 rows, the smallest request the chunk pipeline takes, and instead of asserting identical
answers counts the device answers that differ from torch's fp32 ones, with the float64 logit margin of each row.
"""
import argparse
import json
import sys
import time
from pathlib import Path
from typing import List

import numpy as np
import pandas as pd

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def build_app(predictor_body):
    from fastapi import FastAPI
    from sklearn.datasets import load_digits
    from sklearn.linear_model import LogisticRegression

    from unionml_b200 import Dataset, Model, ModelArtifact

    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    m = Model(name="digits_classifier", init=LogisticRegression, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return load_digits(as_frame=True).frame

    @m.predictor
    def predictor(estimator: LogisticRegression, features: pd.DataFrame) -> List[float]:
        return predictor_body(estimator, features)

    zz = np.load(ROOT / "tests" / "golden" / "digits_lr.npz")
    est = LogisticRegression()
    est.coef_, est.intercept_, est.classes_, est.n_features_in_ = zz["coef"], zz["intercept"], zz["classes"], 64
    m.artifact = ModelArtifact(est)
    app = FastAPI()
    m.serve(app)
    return app, est


def build_mlp_app(predictor_body):
    import torch
    import torch.nn as nn
    import torch.nn.functional as F
    from fastapi import FastAPI
    from sklearn.datasets import load_digits

    from unionml_b200 import Dataset, Model, ModelArtifact

    class PytorchModel(nn.Module):  # tests/integration/pytorch_app/quickstart.py:14-24
        def __init__(self, in_dims, hidden_dims, out_dims):
            super().__init__()
            self.layers = nn.Sequential(nn.Linear(in_dims, hidden_dims), nn.ReLU(), nn.Linear(hidden_dims, out_dims))

        def forward(self, features):
            return F.softmax(self.layers(features), dim=1)

    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    m = Model(name="quickstart_mlp", init=PytorchModel, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return load_digits(as_frame=True).frame

    @m.predictor
    def predictor(module: PytorchModel, features: pd.DataFrame) -> List[float]:
        return predictor_body(module, features)

    torch.manual_seed(0)
    module = PytorchModel(64, 32, 10)
    m.artifact = ModelArtifact(module)
    app = FastAPI()
    m.serve(app)
    return app, module


def drive(app, feats, n_requests):
    from fastapi.testclient import TestClient

    lat, answers = [], []
    with TestClient(app) as client:
        for i in range(n_requests + 30):
            body = {"features": feats.sample(32, random_state=i).to_dict(orient="records")}
            t0 = time.perf_counter()
            r = client.post("/predict", json=body)
            dt = time.perf_counter() - t0
            assert r.status_code == 200 and len(r.json()) == 32
            if i >= 30:
                lat.append(dt * 1e3)
                answers.append(r.json())
    return lat, answers


def call_latency(fn, n=2000):
    for _ in range(100):
        fn()
    out = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e6)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=1000)
    ap.add_argument("--app", default="linear", choices=["linear", "mlp"])
    args = ap.parse_args()
    if args.app == "mlp":
        return main_mlp(args)
    from sklearn.datasets import load_digits

    from unionml_b200.engine import as_feature_array, get_engine
    from unionml_b200.predictors import device_model, linear_argmax

    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]]
    app_gpu, est = build_app(linear_argmax)
    app_cpu, est_cpu = build_app(lambda estimator, features: [float(x) for x in estimator.predict(features)])
    est_cpu.feature_names_in_ = np.asarray(feats.columns, dtype=object)
    lat_gpu, ans_gpu = drive(app_gpu, feats, args.requests)
    lat_cpu, ans_cpu = drive(app_cpu, feats, args.requests)
    assert ans_gpu == ans_cpu, "device and CPU apps must answer identically"
    sample = feats.sample(32, random_state=0)
    est.feature_names_in_ = np.asarray(sample.columns, dtype=object)
    pred_gpu = call_latency(lambda: linear_argmax(est, sample))
    pred_cpu = call_latency(lambda: [float(x) for x in est_cpu.predict(sample)], 500)
    eng = get_engine()
    dm = device_model(est, eng)
    arr = as_feature_array(sample)
    engine_call = call_latency(lambda: eng.predict_host(dm, arr, exact=True))
    q = lambda v, p: float(np.percentile(v, p))  # noqa: E731
    print(json.dumps({
        "config": "cfg4 FastAPI /predict batch=32 (in-process ASGI client), device app vs the reference-shaped CPU app",
        "requests": len(lat_gpu),
        "device_app": {"p50_ms": q(lat_gpu, 50), "p99_ms": q(lat_gpu, 99)},
        "cpu_app": {"p50_ms": q(lat_cpu, 50), "p99_ms": q(lat_cpu, 99)},
        "answers_identical": True,
        "predictor_call_us": {"device_p50": q(pred_gpu, 50), "device_p99": q(pred_gpu, 99),
                              "sklearn_cpu_p50": q(pred_cpu, 50), "sklearn_cpu_p99": q(pred_cpu, 99)},
        "engine_predict_host_call_us": {"p50": q(engine_call, 50), "p99": q(engine_call, 99),
                                        "what": "uml_linear_predict_host on the 32 x 64 float64 block: pinned request buffer, one CUDA graph (H2D, linear_small_kernel, D2H), sync"},
    }), flush=True)


def torch_predictor(module, features):  # the quickstart predictor as written (quickstart.py:31-32, 68-70)
    import torch

    return [float(x) for x in module(torch.from_numpy(features.values).float()).argmax(1)]


def main_mlp(args):
    from sklearn.datasets import load_digits

    from oracle import mlp as omlp
    from unionml_b200.engine import as_feature_array, get_engine
    from unionml_b200.predictors import device_mlp, mlp_argmax

    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]]
    app_gpu, module = build_mlp_app(mlp_argmax)
    app_torch, module_torch = build_mlp_app(torch_predictor)
    lat_gpu, ans_gpu = drive(app_gpu, feats, args.requests)
    lat_torch, ans_torch = drive(app_torch, feats, args.requests)
    w = [t.detach().numpy() for t in (module.layers[0].weight, module.layers[0].bias, module.layers[2].weight,
                                      module.layers[2].bias)]
    differ, margins = 0, []
    for k, (a, b) in enumerate(zip(ans_gpu, ans_torch)):
        rows = [j for j in range(32) if a[j] != b[j]]
        if rows:
            x = feats.sample(32, random_state=30 + k).values[rows]  # drive() times requests 30.. onwards
            differ += len(rows)
            margins += omlp.logit_margin_f64(x, *w).tolist()
    assert all(mg < 1e-4 for mg in margins), "a device answer differs from torch outside torch's fp32 rounding noise"
    sample = feats.sample(32, random_state=0)
    pred_gpu = call_latency(lambda: mlp_argmax(module, sample))
    pred_torch = call_latency(lambda: torch_predictor(module_torch, sample), 500)
    eng = get_engine()
    dm = device_mlp(module, eng)
    arr32 = as_feature_array(sample)
    arr65 = as_feature_array(feats.sample(65, random_state=0))
    assert eng.predict_mlp_host(dm, arr32)[1]["path"] == 4 and eng.predict_mlp_host(dm, arr65)[1]["path"] != 4
    engine32 = call_latency(lambda: eng.predict_mlp_host(dm, arr32, exact=True))
    engine65 = call_latency(lambda: eng.predict_mlp_host(dm, arr65, exact=True))
    q = lambda v, p: float(np.percentile(v, p))  # noqa: E731
    print(json.dumps({
        "config": "FastAPI /predict batch=32 (in-process ASGI client), torch quickstart app: device predictor vs the torch predictor",
        "device": eng.info["name"],
        "requests": len(lat_gpu),
        "device_app": {"p50_ms": q(lat_gpu, 50), "p99_ms": q(lat_gpu, 99)},
        "torch_app": {"p50_ms": q(lat_torch, 50), "p99_ms": q(lat_torch, 99)},
        "answers_differing_from_torch_fp32": differ,
        "max_f64_logit_margin_of_differing_rows": max(margins) if margins else None,
        "predictor_call_us": {"device_p50": q(pred_gpu, 50), "device_p99": q(pred_gpu, 99),
                              "torch_cpu_p50": q(pred_torch, 50), "torch_cpu_p99": q(pred_torch, 99)},
        "engine_predict_mlp_host_call_us": {
            "rows32_p50": q(engine32, 50), "rows32_p99": q(engine32, 99),
            "rows65_p50": q(engine65, 50), "rows65_p99": q(engine65, 99),
            "what": "uml_mlp_predict_host on a 32 x 64 float64 block (online route: pinned request buffer, one CUDA graph "
                    "of mlp_small_kernel, sync) and on 65 rows (chunk pipeline: H2D, stage_convert, tile kernel, fp64 "
                    "re-score, D2H, sync)"},
    }), flush=True)


if __name__ == "__main__":
    main()
