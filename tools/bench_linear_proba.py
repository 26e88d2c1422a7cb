"""float64 class probabilities of the linear predictor against its other outputs, on one GPU (one JSON line).

    python tools/bench_linear_proba.py [--rows 10000000] [--warmup 3] [--iters 10] [--runs 5] [--host-rows 10000000]

cfg 2 shape: 10M x 64 -> 10, bench.py's digits rows (integers 0..16) staged as fp32.  Five routes on the same resident
batch, each writing into a device buffer, timed in alternation (every run times every route `iters` times):
  proba_f32      uml_linear_predict_proba: fp32 scores and expf, float32 result (40 B per row written);
  proba_f64      uml_linear_predict_proba_f64: float64 scores with the softmax epilogue (80 B per row written, path 7);
  log_proba_f64  the same with log_proba = 1;
  scores_f64     uml_linear_decision_function (80 B per row, path 6);
  labels_exact   uml_linear_predict in EXACT mode (4 B per row, path 1; it reads the batch's fp16 copy, 2 B per
                 feature, which staging keeps for these integer rows).
kernel_ms: CUDA events on the engine's stream around the call (the counter reset and the kernel; no copy, the outputs
stay on the device); call_ms: the host clock around the call and a synchronise.  Each is the median over the runs of
the per-run medians; the per-run medians are listed beside it.  Host route: a 10M x 64 float64 pandas frame (pageable,
feature-major) through uml_linear_predict_proba_f64_host, next to scikit-learn's predict_proba on the same frame on this
machine's host cores, alternated the same way.  The card's name, power limit and SM clock come from a read-only
nvidia-smi query in the same process.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.splitlines()[0].split(","))))
    except Exception as e:  # the numbers below are still printed; the card is then unknown
        return {"error": repr(e)}


def med(runs):
    return {"median": round(statistics.median(runs), 4), "runs": [round(t, 4) for t in runs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--host-rows", type=int, default=10_000_000)
    args = ap.parse_args()

    import torch

    from bench import digits_rows
    from unionml_b200.engine import Engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_linear_proba: needs a CUDA device")
    z = np.load(ROOT / "tests" / "golden" / "digits_lr.npz")
    coef, intercept = z["coef"], z["intercept"]
    eng = Engine(0)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)  # the events below time the engine's own work on this stream
    out = {"card": card(), "rows": args.rows, "features": 64, "classes": 10, "runs": args.runs, "iters": args.iters,
           "resident": {}}

    N, F, C = args.rows, 64, 10
    m = eng.load_linear(coef, intercept)
    X = np.empty((N, F), dtype=np.uint8)
    digits_rows(0, N, X)
    b = eng.stage(X.astype(np.float32))
    del X
    p32 = torch.empty((N, C), dtype=torch.float32, device="cuda")
    p64 = torch.empty((N, C), dtype=torch.float64, device="cuda")
    labels = torch.empty(N, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    routes = {
        "proba_f32": lambda: eng.predict_proba(m, b, out_device_ptr=p32.data_ptr()),
        "proba_f64": lambda: eng.predict_proba_f64(m, b, out_device_ptr=p64.data_ptr()),
        "log_proba_f64": lambda: eng.predict_proba_f64(m, b, log=True, out_device_ptr=p64.data_ptr()),
        "scores_f64": lambda: eng.decision_function(m, b, out_device_ptr=p64.data_ptr()),
        "labels_exact": lambda: eng.predict(m, b, exact=True, out_device_ptr=labels.data_ptr()),
    }
    written = {"proba_f32": 4 * C, "proba_f64": 8 * C, "log_proba_f64": 8 * C, "scores_f64": 8 * C, "labels_exact": 4}
    # every route reads the fp32 rows except the labels, which read the batch's fp16 copy when staging kept one
    _, st = eng.predict(m, b, exact=True, out_device_ptr=labels.data_ptr(), want_stats=True)
    read = {k: 4 * F for k in routes}
    read["labels_exact"] = (st.get("x_read_bytes") or 4) * F
    kern = {k: [] for k in routes}
    call = {k: [] for k in routes}
    for name, fn in routes.items():  # warm every route (module load, shared-memory attribute, scratch buffers)
        for _ in range(args.warmup):
            fn()
        eng.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.runs):
        for name, fn in routes.items():
            ks, cs = [], []
            for _ in range(args.iters):
                eng.synchronize()
                t0 = time.perf_counter()
                e0.record(stream)
                fn()
                e1.record(stream)
                eng.synchronize()
                cs.append((time.perf_counter() - t0) * 1e3)
                e1.synchronize()
                ks.append(e0.elapsed_time(e1))
            kern[name].append(statistics.median(ks))
            call[name].append(statistics.median(cs))
    for name in routes:
        km = statistics.median(kern[name])
        out["resident"][name] = {"kernel_ms": med(kern[name]), "call_ms": med(call[name]),
                                 "bytes_per_row": read[name] + written[name],
                                 "gb_per_s": round(N * (read[name] + written[name]) / (km * 1e-3) / 1e9, 1)}
        print(f"{name}: kernel {km:.3f} ms, call {statistics.median(call[name]):.3f} ms", file=sys.stderr)
    # the float64 probabilities of these rows against numpy on a slice (a sanity check of what was timed)
    eng.predict_proba_f64(m, b, out_device_ptr=p64.data_ptr())
    eng.synchronize()
    Xs = np.empty((100_000, F), dtype=np.uint8)
    digits_rows(0, 100_000, Xs)
    s = Xs.astype(np.float64) @ coef.T + intercept
    e = np.exp(s - s.max(axis=1, keepdims=True))
    out["resident"]["proba_f64"]["max_abs_err_vs_numpy"] = float(np.max(np.abs(p64[:100_000].cpu().numpy()
                                                                                - e / e.sum(axis=1, keepdims=True))))
    b.free()
    del p32, p64, labels
    torch.cuda.empty_cache()

    # host route: a 10M x 64 float64 pandas frame (pageable, feature-major), GPU against scikit-learn on the host cores
    import pandas as pd
    from sklearn.linear_model import LogisticRegression

    Nh = args.host_rows
    Xh = np.empty((Nh, F), dtype=np.uint8)
    digits_rows(0, Nh, Xh)
    frame = pd.DataFrame(Xh.astype(np.float64) / 16.0 + 2.0**-30)  # float64 values that are not fp32 values
    del Xh
    est = LogisticRegression()
    est.coef_, est.intercept_, est.classes_ = coef, intercept, z["classes"]
    est.n_features_in_ = F
    gpu_s, cpu_s, st = [], [], None
    eng.predict_proba_f64_host(m, frame.iloc[:100_000])  # warm the pipeline's buffers
    for _ in range(args.runs):
        t0 = time.perf_counter()
        got, st = eng.predict_proba_f64_host(m, frame)
        gpu_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        want = est.predict_proba(frame)
        cpu_s.append(time.perf_counter() - t0)
    out["host"] = {"rows": Nh, "frame": "float64 pandas DataFrame, pageable, feature-major",
                   "gpu_s": med(gpu_s), "sklearn_s": med(cpu_s),
                   "speedup": round(statistics.median(cpu_s) / statistics.median(gpu_s), 2),
                   "path": st["path"], "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                   "max_abs_err_vs_sklearn": float(np.max(np.abs(got - want))),
                   "host_cpus": len(os.sched_getaffinity(0))}
    print(f"host: gpu {out['host']['gpu_s']['median']} s, sklearn {out['host']['sklearn_s']['median']} s", file=sys.stderr)
    eng.set_stream(None)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
