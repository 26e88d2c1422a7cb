"""The MLP predictor's class probabilities and top-k from host rows (one JSON line; not part of the driver contract).

    python tools/bench_mlp_host_outputs.py [--calls 1000] [--rows 10000000] [--k 3]

The golden torch-quickstart network (64 -> 32 -> 10, tests/golden/mlp_64_32_10.npz) on digits-like rows (integers
0..16, float64, as a pandas frame):
  * online: engine-call p50 / p99 of 1-row and 32-row requests (what the quickdraw template's /predict sends) for
    probabilities and top-k through the host routes (Engine.predict_mlp_proba_host / predict_mlp_topk_host: one
    float64 kernel replayed as a CUDA graph), next to the labels' online call and the earlier route, stage + resident
    call + free (Engine.stage, predict_mlp_proba / predict_mlp_topk, Batch.free).
  * frame: one --rows x 64 float64 pandas frame, probabilities and top-k through the chunk pipeline, the earlier
    stage + resident route, and torch on the CPU (module(x) and torch.topk of it, on torch's default threads).
Each timed call ends in a synchronise (the engine calls are synchronous).
"""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import pandas as pd

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tools.bench_mlp_topk import card  # noqa: E402


def pct(ts):
    ts = sorted(ts)
    return {"p50_us": round(1e6 * statistics.median(ts), 1), "p99_us": round(1e6 * ts[int(0.99 * (len(ts) - 1))], 1)}


def timed(fn, calls, warmup=20):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=3)
    args = ap.parse_args()

    import torch

    from bench import digits_rows
    from unionml_b200.engine import Engine

    g = np.load(ROOT / "tests" / "golden" / "mlp_64_32_10.npz")
    w = (g["w1"], g["b1"], g["w2"], g["b2"])
    eng = Engine(0)
    m = eng.load_mlp(*w)
    k = args.k
    cols = [f"pixel_{i}" for i in range(64)]
    out = {"card": card(), "k": k, "calls": args.calls}

    def staged(fn):
        def call(X):
            b = eng.stage(X.to_numpy(), keep_f64=False)
            try:
                return fn(b)
            finally:
                b.free()
        return call

    old_proba = staged(lambda b: eng.predict_mlp_proba(m, b))
    old_topk = staged(lambda b: eng.predict_mlp_topk(m, b, k, exact=True))
    online = {}
    for rows in (1, 32):
        X = pd.DataFrame(np.random.default_rng(rows).integers(0, 17, size=(rows, 64)).astype(np.float64), columns=cols)
        assert eng.predict_mlp_proba_host(m, X)[1]["path"] == 4 and eng.predict_mlp_topk_host(m, X, k)[2]["path"] == 4
        online[f"{rows}_rows"] = {
            "labels_online": pct(timed(lambda: eng.predict_mlp_host(m, X), args.calls)),
            "proba_online": pct(timed(lambda: eng.predict_mlp_proba_host(m, X), args.calls)),
            "proba_stage_resident": pct(timed(lambda: old_proba(X), args.calls)),
            f"top{k}_online": pct(timed(lambda: eng.predict_mlp_topk_host(m, X, k), args.calls)),
            f"top{k}_stage_resident": pct(timed(lambda: old_topk(X), args.calls)),
        }
    out["online"] = online

    N = args.rows
    X8 = np.empty((N, 64), dtype=np.uint8)
    digits_rows(0, N, X8)
    frame = pd.DataFrame(X8.astype(np.float64), columns=cols)
    del X8

    def once(fn):
        fn()  # warm: scratch and pinned buffers grow on the first call
        t0 = time.perf_counter()
        r = fn()
        return time.perf_counter() - t0, r

    t_pp, (pp, st_p) = once(lambda: eng.predict_mlp_proba_host(m, frame))
    t_pt, (pi, _, st_t) = once(lambda: eng.predict_mlp_topk_host(m, frame, k))
    t_op, (op, _) = once(lambda: old_proba(frame))
    t_ot, (oi, _, _) = once(lambda: old_topk(frame))
    assert np.array_equal(pp.view(np.uint32), op.view(np.uint32)) and np.array_equal(pi, oi)
    del pp, op, pi, oi
    module = torch.nn.Sequential(torch.nn.Linear(64, 32), torch.nn.ReLU(), torch.nn.Linear(32, 10))
    with torch.no_grad():
        for p, v in zip(module.parameters(), w):
            p.copy_(torch.from_numpy(v))
        t0 = time.perf_counter()
        probs = torch.softmax(module(torch.from_numpy(frame.values).float()), dim=1)
        t_cpu_p = time.perf_counter() - t0
        t0 = time.perf_counter()
        torch.topk(torch.softmax(module(torch.from_numpy(frame.values).float()), dim=1), k)
        t_cpu_t = time.perf_counter() - t0
    del probs
    out["frame"] = {
        "rows": N, "path_proba": st_p["path"], "path_topk": st_t["path"], "torch_threads": torch.get_num_threads(),
        "proba_pipeline_s": round(t_pp, 4), "proba_stage_resident_s": round(t_op, 4), "proba_torch_cpu_s": round(t_cpu_p, 4),
        f"top{k}_pipeline_s": round(t_pt, 4), f"top{k}_stage_resident_s": round(t_ot, 4),
        f"top{k}_torch_cpu_s": round(t_cpu_t, 4),
    }
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
