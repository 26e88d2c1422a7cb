"""Top-3 classes with probabilities against labels and full probabilities of the MLP predictor at the cfg 5 shape, on
one GPU (one JSON line).

    python tools/bench_mlp_topk.py [--rows 10000000] [--warmup 5] [--iters 30]

The batch is bench.py's cfg 5 batch: 10M x 64 digits-domain rows (integers 0..16, chunk k = default_rng(k)) and the
64 -> 32 -> 10 module of torch.manual_seed(0); then the same shape on standard-normal rows.  In one process the script
alternates three calls, all writing to device buffers: the EXACT top-3 with probabilities (uml_mlp_predict_topk), the
EXACT labels (uml_mlp_predict) and the full probabilities (uml_mlp_predict_proba).  Times are the engine's CUDA events
(stats): kernel_ms brackets the scoring kernel, recheck_ms the float64 re-score behind it; medians and min-max over
the timed launches.  The flagged-row counts of the top-3 guard and of the label guard are reported side by side.  The
card's name, power limit and SM clock come from a read-only nvidia-smi query.
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


def summary(ts):
    return {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--k", type=int, default=3)
    args = ap.parse_args()

    import torch
    import torch.nn as nn

    from bench import digits_rows
    from unionml_b200.engine import Engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp_topk: needs a CUDA device")
    torch.manual_seed(0)
    module = nn.Sequential(nn.Linear(64, 32), nn.ReLU(), nn.Linear(32, 10))  # PytorchModel(64, 32, 10)'s layers
    w = [t.detach().numpy() for t in (module[0].weight, module[0].bias, module[2].weight, module[2].bias)]
    eng = Engine(0)
    m = eng.load_mlp(*w)
    N, F, C, k = args.rows, 64, 10, args.k
    X = np.empty((N, F), dtype=np.uint8)
    digits_rows(0, N, X)
    batches = {"path5_digits": eng.stage(X)}
    del X
    g = torch.Generator(device="cuda").manual_seed(0)
    Xn = torch.randn((N, F), generator=g, device="cuda", dtype=torch.float32)
    batches["path3_normal"] = eng.wrap_device(Xn.data_ptr(), N, F, keepalive=Xn)
    labels = torch.empty(N, dtype=torch.int32, device="cuda")
    idx = torch.empty((N, k), dtype=torch.int32, device="cuda")
    topp = torch.empty((N, k), dtype=torch.float32, device="cuda")
    proba = torch.empty((N, C), dtype=torch.float32, device="cuda")

    out = {"card": card(), "rows": N, "features": F, "classes": C, "k": k, "iters": args.iters, "routes": {}}
    for name, b in batches.items():
        t = {"topk_kernel": [], "topk_rescore": [], "topk_total": [], "labels_kernel": [], "labels_rescore": [],
             "labels_total": [], "proba_kernel": []}
        paths, flagged = set(), {}
        for i in range(args.warmup + args.iters):
            _, _, st = eng.predict_mlp_topk(m, b, k, exact=True, idx_device_ptr=idx.data_ptr(),
                                            proba_device_ptr=topp.data_ptr())
            _, sl = eng.predict_mlp(m, b, exact=True, out_device_ptr=labels.data_ptr(), want_stats=True)
            _, sp = eng.predict_mlp_proba(m, b, out_device_ptr=proba.data_ptr(), want_stats=True)
            paths.add((st["path"], sl["path"], sp["path"]))
            flagged = {"topk": st["n_flagged"], "labels": sl["n_flagged"]}
            if i >= args.warmup:
                t["topk_kernel"].append(st["kernel_ms"])
                t["topk_rescore"].append(st["recheck_ms"])
                t["topk_total"].append(st["kernel_ms"] + st["recheck_ms"])
                t["labels_kernel"].append(sl["kernel_ms"])
                t["labels_rescore"].append(sl["recheck_ms"])
                t["labels_total"].append(sl["kernel_ms"] + sl["recheck_ms"])
                t["proba_kernel"].append(sp["kernel_ms"])
        route = {"paths": sorted(paths), "n_flagged": flagged, "ms": {key: summary(v) for key, v in t.items()}}
        route["topk_over_labels"] = round(route["ms"]["topk_total"]["median"] / route["ms"]["labels_total"]["median"], 3)
        out["routes"][name] = route
        print(f"{name}: top-{k} {route['ms']['topk_total']['median']:.3f} ms, labels {route['ms']['labels_total']['median']:.3f} ms, "
              f"proba {route['ms']['proba_kernel']['median']:.3f} ms, flagged {flagged}, paths {route['paths']}", file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
