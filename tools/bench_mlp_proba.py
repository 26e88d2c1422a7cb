"""Class probabilities against labels of the MLP predictor at the cfg 5 shape, on one GPU (one JSON line).

    python tools/bench_mlp_proba.py [--rows 10000000] [--warmup 5] [--iters 30]

The batch is bench.py's cfg 5 batch: 10M x 64 digits-domain rows (integers 0..16, chunk k = default_rng(k)) and the
64 -> 32 -> 10 module of torch.manual_seed(0).  In one process the script alternates the FAST argmax kernel
(uml_mlp_predict) and the probability kernel (uml_mlp_predict_proba), both writing to device buffers: first on
those rows (tensor cores, path 5), then on standard-normal rows (CUDA cores, path 3).  Times are the engine's CUDA
events around the kernel (stats kernel_ms), medians over the timed launches.  Bytes moved: 4 F per row read, 4 C per
row written for probabilities and 4 for labels, against MEASURED_PEAKS.json's read ceiling when it exists (written by
tools/linear_probe.sh), else against the 3.35 TB/s of the H100 SXM data sheet.  The card's name, power limit and SM
clock come from a read-only nvidia-smi query.
"""
import argparse
import json
import statistics
import subprocess
import sys
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()

    import torch
    import torch.nn as nn

    from bench import digits_rows
    from unionml_b200.engine import Engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp_proba: needs a CUDA device")
    torch.manual_seed(0)
    module = nn.Sequential(nn.Linear(64, 32), nn.ReLU(), nn.Linear(32, 10))  # PytorchModel(64, 32, 10)'s layers
    w = [t.detach().numpy() for t in (module[0].weight, module[0].bias, module[2].weight, module[2].bias)]
    eng = Engine(0)
    m = eng.load_mlp(*w)
    N, F, C = args.rows, 64, 10
    X = np.empty((N, F), dtype=np.uint8)
    digits_rows(0, N, X)
    batches = {"path5_digits": eng.stage(X)}
    del X
    g = torch.Generator(device="cuda").manual_seed(0)
    Xn = torch.randn((N, F), generator=g, device="cuda", dtype=torch.float32)
    batches["path3_normal"] = eng.wrap_device(Xn.data_ptr(), N, F, keepalive=Xn)
    labels = torch.empty(N, dtype=torch.int32, device="cuda")
    proba = torch.empty((N, C), dtype=torch.float32, device="cuda")
    ceiling, ceiling_src = read_ceiling()

    out = {"card": card(), "rows": N, "features": F, "classes": C, "iters": args.iters, "ceiling_gbs": ceiling,
           "ceiling": ceiling_src, "routes": {}}
    for name, b in batches.items():
        times = {"labels": [], "proba": []}
        paths = set()
        for i in range(args.warmup + args.iters):
            _, sl = eng.predict_mlp(m, b, exact=False, out_device_ptr=labels.data_ptr(), want_stats=True)
            _, sp = eng.predict_mlp_proba(m, b, out_device_ptr=proba.data_ptr(), want_stats=True)
            paths.add((sl["path"], sp["path"]))
            if i >= args.warmup:
                times["labels"].append(sl["kernel_ms"])
                times["proba"].append(sp["kernel_ms"])
        route = {"paths": sorted(paths)}
        for kind, ts in times.items():
            ms = statistics.median(ts)
            moved = N * (4 * F + (4 * C if kind == "proba" else 4))
            route[kind] = {"kernel_ms": round(ms, 4), "kernel_ms_min": round(min(ts), 4), "kernel_ms_max": round(max(ts), 4),
                           "rows_per_s": round(N / (ms * 1e-3)), "bytes": moved,
                           "gb_per_s": round(moved / (ms * 1e-3) / 1e9, 1),
                           "of_ceiling": round(moved / (ms * 1e-3) / 1e9 / ceiling, 3)}
        route["proba_over_labels"] = round(route["proba"]["kernel_ms"] / route["labels"]["kernel_ms"], 3)
        out["routes"][name] = route
        print(f"{name}: labels {route['labels']['kernel_ms']:.3f} ms, proba {route['proba']['kernel_ms']:.3f} ms "
              f"(x{route['proba_over_labels']}), paths {route['paths']}", file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
