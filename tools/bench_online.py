"""cfg 4 of BASELINE.json: FastAPI /predict online serving, batch = 32, p50 / p99 latency on 1 x H100 - with the
reference-shaped CPU predictor served through the SAME app beside it (one JSON line; not part of the driver contract).

    python tools/bench_online.py [--requests 1000]

Both apps are `unionml_b200.Model.serve(FastAPI())` (mirror of unionml:unionml/fastapi.py:15-70) driven by the
in-process ASGI TestClient with 1 000 POSTs of digits.frame[features].sample(32, random_state=i) records (SURVEY.md 8d):
  * device : @model.predictor = unionml_b200.predictors.linear_argmax  (small-batch float64 kernel, CUDA graph replay)
  * cpu    : @model.predictor = [float(x) for x in estimator.predict(features)]  (unionml:README.md:87-92)
and the predictor call alone is timed for both (what the device path changes inside a request).
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
    args = ap.parse_args()
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


if __name__ == "__main__":
    main()
