"""float64 decision_function scores against EXACT labels of the linear predictor, on one GPU (one JSON line).

    python tools/bench_decision_function.py [--rows 10000000] [--warmup 5] [--iters 30] [--host-rows 10000000]

Resident routes, timed alternately in one process with the engine's CUDA events around the kernel (stats kernel_ms;
medians, min-max beside them):
  cfg2      10M x 64 -> 10, bench.py's digits rows (integers 0..16) as fp32: the scores kernel (uml_linear_decision_function,
            path 6) against the EXACT label kernel (uml_linear_predict, path 1), both into device buffers;
  cfg2_f64  the same rows with a float64 copy (UML_STAGE_KEEP_F64 on rows that are not fp32 values): scores read the
            copy (512 B per row), labels the fp32 rows;
  cfg3      784 -> 10 (pixels / 255 as fp32), the largest row count whose fp32 rows and scores fit in half the free memory.
Bytes per launch: F x 4 (or 8) read + C x 8 written for scores, F x 4 read + 4 written for labels, against
MEASURED_PEAKS.json's read ceiling when it exists (written by tools/linear_probe.sh), else the 3.35 TB/s of the H100
SXM data sheet (the JSON says which).  Host route: a 10M x 64 float64 pandas frame (pageable, feature-major) through
uml_linear_decision_function_host, next to scikit-learn's decision_function on the same frame on this machine's host
cores.  The card's name, power limit and SM clock come from a read-only nvidia-smi query.
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


def read_ceiling():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        return float(json.loads(p.read_text())["hbm_gbs"]), "measured read ceiling (MEASURED_PEAKS.json)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not measured"


def summary(ts, n, moved, ceiling):
    ms = statistics.median(ts)
    return {"kernel_ms": round(ms, 4), "kernel_ms_min": round(min(ts), 4), "kernel_ms_max": round(max(ts), 4),
            "rows_per_s": round(n / (ms * 1e-3)), "bytes": moved, "gb_per_s": round(moved / (ms * 1e-3) / 1e9, 1),
            "of_ceiling": round(moved / (ms * 1e-3) / 1e9 / ceiling, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--host-rows", type=int, default=10_000_000)
    ap.add_argument("--host-iters", type=int, default=3)
    args = ap.parse_args()

    import torch

    from bench import digits_rows
    from unionml_b200.engine import Engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_decision_function: needs a CUDA device")
    z = np.load(ROOT / "tests" / "golden" / "digits_lr.npz")
    coef, intercept = z["coef"], z["intercept"]
    eng = Engine(0)
    ceiling, ceiling_src = read_ceiling()
    out = {"card": card(), "iters": args.iters, "ceiling_gbs": ceiling, "ceiling": ceiling_src, "routes": {}}

    def alternate(name, m, batch, n, F, C, read_bytes):
        labels = torch.empty(n, dtype=torch.int32, device="cuda")
        scores = torch.empty((n, C), dtype=torch.float64, device="cuda")
        times = {"scores": [], "labels": []}
        paths = set()
        for i in range(args.warmup + args.iters):
            _, ss = eng.decision_function(m, batch, out_device_ptr=scores.data_ptr(), want_stats=True)
            _, sl = eng.predict(m, batch, exact=True, out_device_ptr=labels.data_ptr(), want_stats=True)
            paths.add((ss["path"], sl["path"]))
            if i >= args.warmup:
                times["scores"].append(ss["kernel_ms"])
                times["labels"].append(sl["kernel_ms"])
        route = {"rows": n, "features": F, "classes": C, "paths": sorted(paths),
                 "scores": summary(times["scores"], n, n * (read_bytes + 8 * C), ceiling),
                 "labels_exact": summary(times["labels"], n, n * (4 * F + 4), ceiling)}
        route["scores_over_labels"] = round(route["scores"]["kernel_ms"] / route["labels_exact"]["kernel_ms"], 3)
        out["routes"][name] = route
        print(f"{name}: scores {route['scores']['kernel_ms']:.3f} ms ({route['scores']['of_ceiling']} of ceiling), "
              f"labels {route['labels_exact']['kernel_ms']:.3f} ms, paths {route['paths']}", file=sys.stderr)
        del labels, scores
        torch.cuda.empty_cache()

    # cfg 2: fp32 digits rows, then the same rows with a float64 copy
    N, F, C = args.rows, 64, 10
    m = eng.load_linear(coef, intercept)
    X = np.empty((N, F), dtype=np.uint8)
    digits_rows(0, N, X)
    b = eng.stage(X)
    alternate("cfg2", m, b, N, F, C, 4 * F)
    b.free()
    # a float64 frame whose fp32 cast is lossy keeps its float64 copy: digits + 2^-30 (the scores read 8 B per feature)
    Xd = X.astype(np.float64) + 2.0**-30
    del X
    b = eng.stage(Xd, keep_f64=True)
    assert not b.lossless
    alternate("cfg2_f64", m, b, N, F, C, 8 * F)
    b.free()
    del Xd

    # cfg 3: 784 -> 10 on pixels / 255 as fp32, the largest row count that fits in half the free memory
    F3 = 784
    rng = np.random.default_rng(0)
    m3 = eng.load_linear(rng.standard_normal((C, F3)) * 0.01, rng.standard_normal(C))
    free, _ = torch.cuda.mem_get_info()
    n3 = int(min(args.rows, 0.5 * free // (4 * F3 + 8 * C + 4)))
    g = torch.Generator(device="cuda").manual_seed(0)
    x3 = torch.randint(0, 256, (n3, F3), generator=g, device="cuda", dtype=torch.int32).to(torch.float32).div_(255.0)
    torch.cuda.synchronize()  # written on torch's stream; the engine runs on its own
    b3 = eng.wrap_device(x3.data_ptr(), n3, F3, keepalive=x3)
    alternate("cfg3", m3, b3, n3, F3, C, 4 * F3)
    b3.free()
    del x3
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
    gpu_s, cpu_s, st = [], [], None
    for _ in range(args.host_iters):
        t0 = time.perf_counter()
        got, st = eng.decision_function_host(m, frame)
        gpu_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        want = est.decision_function(frame)
        cpu_s.append(time.perf_counter() - t0)
    scale = np.abs(frame.to_numpy()) @ np.abs(coef).T + np.abs(intercept)
    out["host"] = {"rows": Nh, "features": F, "frame": "float64 pandas DataFrame, pageable, feature-major",
                   "gpu_s": round(statistics.median(gpu_s), 4), "gpu_s_all": [round(t, 4) for t in gpu_s],
                   "sklearn_s": round(statistics.median(cpu_s), 4), "sklearn_s_all": [round(t, 4) for t in cpu_s],
                   "speedup": round(statistics.median(cpu_s) / statistics.median(gpu_s), 2),
                   "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                   "max_err_over_scale": float(np.max(np.abs(got - want) / scale)),
                   "host_cpus": len(os.sched_getaffinity(0))}
    print(f"host: gpu {out['host']['gpu_s']} s, sklearn {out['host']['sklearn_s']} s", file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
