#!/usr/bin/env python
"""A/B of the linear tile kernel on bench.py's cfg 2 batch: fp32 rows against the batch's compact fp16 copy.

    python tools/ab_compact_rows.py [--probe build/probe/linear_probe.jsonl] [--warmup 5] [--launches 30]

Stages the cfg 2 batch (10M x 64 integers 0..16, bench.digits_rows) and the golden digits model once, then alternates
the two routes of the same batch through UML_B200_COMPACT_ROWS (0: fp32 rows; unset: the fp16 copy), one launch at a
time: the EXACT, uint8-label predict_peers step bench.py times, bracketed by CUDA events on the engine's stream.
Prints one JSON object: per route the median and min-max kernel time, the bytes it reads (4 F and 2 F per row) and
their rate, n_flagged, whether all labels are byte-equal, and the card's name, power limit and SM clock.  With --probe,
the read ceilings over 1.28 GB and 2.56 GB come from tools/linear_probe.sh's output (run it in the same session on
the same card), and each route's share of the ceiling over the bytes it actually reads is reported beside them.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), (v.strip() for v in r.stdout.strip().split(",")))) if r.returncode == 0 else {}


def read_ceilings(path):
    """{bytes: GB/s} of the probe's read_ceiling lines."""
    out = {}
    for line in Path(path).read_text().splitlines():
        if line.startswith("{"):
            r = json.loads(line)
            if r.get("probe") == "read_ceiling":
                out[int(r["bytes"])] = r["hbm_gbs"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--probe", default=None, help="linear_probe.jsonl written by tools/linear_probe.sh in this session")
    ap.add_argument("--warmup", type=int, default=5, help="warm-up pairs")
    ap.add_argument("--launches", type=int, default=30, help="timed launches per route")
    args = ap.parse_args()

    import torch

    from bench import CONFIGS, digits_rows, load_model_arrays
    from unionml_b200.engine import Engine

    cfg = CONFIGS["cfg2"]
    n, F = cfg["rows"], cfg["F"]
    eng = Engine(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    arrs = load_model_arrays(cfg)
    model = eng.load_linear(arrs["coef"], arrs["intercept"], arrs["classes"])
    X = eng.pinned_empty((n, F), np.float32)
    digits_rows(0, n, X)
    batch = eng.stage(X)
    labels = {r: torch.empty(n, dtype=torch.uint8, device="cuda") for r in ("fp32", "fp16")}

    def step(route, want_stats=False):
        if route == "fp32":
            os.environ["UML_B200_COMPACT_ROWS"] = "0"
        else:
            os.environ.pop("UML_B200_COMPACT_ROWS", None)
        return eng.predict_peers(model, batch, [labels[route].data_ptr()], 0, exact=True, want_stats=want_stats,
                                 label_bytes=1)

    stats = {r: step(r, want_stats=True) for r in ("fp32", "fp16")}
    assert stats["fp32"]["x_elem_bytes"] == 4 and stats["fp16"]["x_elem_bytes"] == 2, stats
    equal = bool(torch.equal(labels["fp32"], labels["fp16"]))
    before = card()
    for _ in range(args.warmup):
        step("fp32")
        step("fp16")
    ms = {"fp32": [], "fp16": []}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(args.launches):
        for route in ("fp32", "fp16"):
            ev[0].record(stream)
            step(route)
            ev[1].record(stream)
            ev[1].synchronize()
            ms[route].append(ev[0].elapsed_time(ev[1]))
    after = card()
    os.environ.pop("UML_B200_COMPACT_ROWS", None)
    ceilings = read_ceilings(args.probe) if args.probe else {}

    out = {"rows": n, "features": F, "launches_per_route": args.launches, "warmup_pairs": args.warmup,
           "labels_byte_equal": equal, "card_before": before, "card_after": after, "routes": {}}
    for route, elem in (("fp32", 4), ("fp16", 2)):
        med = statistics.median(ms[route])
        read = n * F * elem
        r = {"x_elem_bytes": elem, "bytes_read": read, "ms_median": med, "ms_min": min(ms[route]),
             "ms_max": max(ms[route]), "gbs_median": read / (med * 1e-3) / 1e9, "n_flagged": stats[route]["n_flagged"],
             "rows_per_s_median": n / (med * 1e-3)}
        ceil = ceilings.get(read)
        if ceil:
            r["read_ceiling_gbs"] = ceil
            r["read_ceiling_ms"] = read / (ceil * 1e9) * 1e3
            r["frac_of_ceiling"] = r["gbs_median"] / ceil
        out["routes"][route] = r
    out["speedup_median"] = out["routes"]["fp32"]["ms_median"] / out["routes"]["fp16"]["ms_median"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
