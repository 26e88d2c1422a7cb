#!/usr/bin/env python
"""Round-2 probes on one GPU (not a bench line): staging-kernel bandwidth, pageable-source H2D rate with and without
the pinned bounce pool, online-path latency (<= 64 rows), and the step time of a 1.25M-row shard (the strong-scaling
share of cfg 2 at 8 GPUs).  Writes gpurun_out/probe_r2.json."""
from __future__ import annotations

import json
import os
import statistics
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def main():
    import pandas as pd
    import torch

    from unionml_b200.engine import Engine

    out = {}
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    z = np.load(ROOT / "tests" / "golden" / "digits_lr.npz")
    model = eng.load_linear(z["coef"], z["intercept"], z["classes"])

    # ---- (1) step time vs rows on the resident path (async, u8 labels): launch overhead at strong-scaling shard sizes
    steps = {}
    for rows in (156_250, 625_000, 1_250_000, 2_500_000, 5_000_000, 10_000_000):
        X = torch.randint(0, 17, (rows, 64), device=dev, dtype=torch.int32).to(torch.float32)
        b = eng.wrap_device(X.data_ptr(), rows, 64, keepalive=X)
        lab = torch.empty(rows, dtype=torch.uint8, device=dev)
        for _ in range(5):
            eng.predict_peers(model, b, [lab.data_ptr()], 0, exact=True, label_bytes=1)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        K = 50
        for _ in range(K):
            eng.predict_peers(model, b, [lab.data_ptr()], 0, exact=True, label_bytes=1)
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / K
        # the same K steps replayed as one CUDA graph
        g_ms = None
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                for _ in range(10):
                    eng.predict_peers(model, b, [lab.data_ptr()], 0, exact=True, label_bytes=1)
            g.replay()
            torch.cuda.synchronize()
            e0.record(stream)
            for _ in range(5):
                g.replay()
            e1.record(stream)
            torch.cuda.synchronize()
            g_ms = e0.elapsed_time(e1) / 50
        except Exception as exc:  # capture not possible: report why
            g_ms = repr(exc)
        torch.cuda.set_stream(stream)
        eng.set_stream(stream.cuda_stream)
        steps[rows] = {"ms_per_step": ms, "graph_ms_per_step": g_ms, "hbm_ms": rows * 256 / 6489.6e9 * 1e3}
        del b, X, lab
    out["step_vs_rows"] = steps

    # ---- (2) pageable float64 frame -> labels: bounce pool on / off
    rows = 4_000_000
    Xf = np.empty((64, rows), dtype=np.float64)
    for k in range(4):
        Xf[:, k * 1_000_000 : (k + 1) * 1_000_000] = np.random.default_rng(k).integers(0, 17, size=(64, 1_000_000))
    frame = pd.DataFrame(Xf.T, columns=[f"pixel_{i}" for i in range(64)], copy=False)
    arr = frame.to_numpy()
    out["frame_to_numpy_strides"] = list(arr.strides)
    res = {}
    for label, env in (("bounce", None), ("driver_staged", "1")):
        if env:
            os.environ["UML_B200_NO_BOUNCE"] = env
        else:
            os.environ.pop("UML_B200_NO_BOUNCE", None)
        ts = []
        for i in range(4):
            t0 = time.perf_counter()
            idx, st = eng.predict_host(model, arr, exact=True)
            dt = time.perf_counter() - t0
            if i:
                ts.append(dt)
        res[label] = {"s": min(ts), "h2d_GBps": st["h2d_bytes"] / min(ts) / 1e9, "rows_per_s": rows / min(ts)}
    os.environ.pop("UML_B200_NO_BOUNCE", None)
    # C-order float32 pageable and pinned, for the link-rate reference
    Xc = np.ascontiguousarray(Xf.T.astype(np.float32))
    for label, a in (("f32_pageable_bounce", Xc),):
        ts = []
        for i in range(4):
            t0 = time.perf_counter()
            idx, st = eng.predict_host(model, a, exact=True)
            dt = time.perf_counter() - t0
            if i:
                ts.append(dt)
        res[label] = {"s": min(ts), "h2d_GBps": st["h2d_bytes"] / min(ts) / 1e9, "rows_per_s": rows / min(ts)}
    Xp = eng.pinned_empty(Xc.shape, np.float32)
    Xp[:] = Xc
    ts = []
    for i in range(4):
        t0 = time.perf_counter()
        idx, st = eng.predict_host(model, Xp, exact=True)
        dt = time.perf_counter() - t0
        if i:
            ts.append(dt)
    res["f32_pinned"] = {"s": min(ts), "h2d_GBps": st["h2d_bytes"] / min(ts) / 1e9, "rows_per_s": rows / min(ts)}
    out["host_sources_4M_rows"] = res

    # ---- (3) API-level: float64 frame -> List[float] through linear_argmax vs the reference predictor on the CPU
    from sklearn.linear_model import LogisticRegression

    from unionml_b200.predictors import linear_argmax

    est = LogisticRegression()
    est.coef_, est.intercept_, est.classes_, est.n_features_in_ = z["coef"], z["intercept"], z["classes"], 64
    est.feature_names_in_ = np.asarray(frame.columns, dtype=object)
    linear_argmax(est, frame.iloc[:100_000])
    t0 = time.perf_counter()
    got = linear_argmax(est, frame)
    t_gpu = time.perf_counter() - t0
    sub = frame.iloc[:1_000_000]
    t0 = time.perf_counter()
    want = [float(x) for x in est.predict(sub)]
    t_cpu = time.perf_counter() - t0
    out["api_frame_to_list"] = {"rows": rows, "gpu_s": t_gpu, "gpu_rows_per_s": rows / t_gpu, "cpu_rows": 1_000_000,
                                "cpu_s": t_cpu, "cpu_rows_per_s": 1_000_000 / t_cpu, "equal_first_million": got[:1_000_000] == want}

    # ---- (4) online path latency: 32-row frames through the predictor
    small = frame.iloc[:32]
    for fn, name in ((lambda: linear_argmax(est, small), "linear_argmax_32"), (lambda: [float(x) for x in est.predict(small)], "sklearn_32")):
        for _ in range(50):
            fn()
        ts = []
        for _ in range(1000):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        ts.sort()
        out[name] = {"p50_us": ts[500] * 1e6, "p99_us": ts[990] * 1e6}
    a32 = small.to_numpy()
    ts = []
    for _ in range(1000):
        t0 = time.perf_counter()
        eng.predict_host(model, a32, exact=True)
        ts.append(time.perf_counter() - t0)
    ts.sort()
    out["engine_predict_host_32"] = {"p50_us": ts[500] * 1e6, "p99_us": ts[990] * 1e6}

    # ---- (5) staging kernels in isolation (device-resident raw chunk -> fp32 rows): launch via stage() of pinned sources
    stg = {}
    rows = 4_000_000
    for name, src in (("featmajor_f64", np.asfortranarray(Xf.T)), ("rowmajor_f64", np.ascontiguousarray(Xf.T))):
        pin = eng.pinned_empty(src.shape, np.float64)
        if name.startswith("feat"):
            pinT = eng.pinned_empty((64, rows), np.float64)
            pinT[:] = Xf
            src_arr = pinT.T
        else:
            pin[:] = src
            src_arr = pin
        ts = []
        for i in range(3):
            t0 = time.perf_counter()
            b = eng.stage(src_arr)
            ts.append(time.perf_counter() - t0)
            b.free()
        stg[name] = {"stage_s": min(ts), "GBps_in": rows * 64 * 8 / min(ts) / 1e9}
    out["stage_calls"] = stg

    # ---- (6) where the time of the MLP drop-in predictor goes (float64 frame -> List[float])
    import torch.nn as nn

    from unionml_b200.engine import get_engine
    from unionml_b200.predictors import device_mlp, mlp_argmax

    zz = np.load(ROOT / "tests" / "golden" / "mlp_64_32_10.npz")
    module = nn.Sequential(nn.Linear(64, 32), nn.ReLU(), nn.Linear(32, 10))
    with torch.no_grad():
        module[0].weight.copy_(torch.from_numpy(zz["w1"])); module[0].bias.copy_(torch.from_numpy(zz["b1"]))
        module[2].weight.copy_(torch.from_numpy(zz["w2"])); module[2].bias.copy_(torch.from_numpy(zz["b2"]))
    mlp_argmax(module, frame.iloc[:100_000])
    ge = get_engine()
    dm = device_mlp(module, ge)
    tt = {}
    for rep in range(2):
        t0 = time.perf_counter(); a = frame.to_numpy(); t1 = time.perf_counter()
        b = ge.stage(a, keep_f64=False); t2 = time.perf_counter()
        idx, _ = ge.predict_mlp(dm, b, exact=True); t3 = time.perf_counter()
        b.free(); t4 = time.perf_counter()
        lst = idx.astype(np.float64).tolist(); t5 = time.perf_counter()
        tt = {"to_numpy": t1 - t0, "stage": t2 - t1, "predict_mlp": t3 - t2, "free": t4 - t3, "astype_tolist": t5 - t4}
    t0 = time.perf_counter(); mlp_argmax(module, frame); tt["mlp_argmax_total"] = time.perf_counter() - t0
    out["mlp_argmax_4M_breakdown_s"] = tt

    Path(ROOT / "gpurun_out").mkdir(exist_ok=True)
    (ROOT / "gpurun_out" / "probe_r2.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
