#!/usr/bin/env python
"""A/B of the linear tile kernel's schedules on bench.py's cfg 2 batch: the tensor-core schedule on the byte copy
(the default; x_read_bytes 1), the tensor-core schedule on the fp16 copy
(UML_B200_COMPACT_ROWS=2 with UML_B200_LINEAR_TC=1, which fails unless a tensor-core schedule runs) and the CUDA-core
fp16 schedule (UML_B200_LINEAR_TC=0).

    python tools/ab_linear_tc.py [--warmup 5] [--launches 30]

Stages the cfg 2 batch and the golden digits model once, alternates the three schedules one launch at a time (the EXACT,
uint8-label predict_peers step bench.py times, bracketed by CUDA events), and prints one JSON object: per schedule the
median and min-max time and n_flagged, whether the labels are byte-equal, the card's name, power limit and SM clock,
and how many rows tier 1 leaves to the fp32 replay.  That count is measured by one untimed call with
UML_B200_TC_REPLAY=0 (every row tier 1 leaves then goes to float64 and counts in n_flagged), and estimated beside it
from float64 scores as a cross-check: rows whose exact top-2 margin is at most kappa A (the tensor-core guard's
threshold; kappa as build_tc_operands computes it) or at most thr A (the fp32 route's; these are the rows it flags, up
to its rounding).
"""
import argparse
import json
import os
import statistics
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

U = 2.0**-24


def thresholds(F):
    """(thr, kappa) of a 64-feature-wide fp16 row: linear_margin_thr and build_tc_operands' factor."""
    thr = float(np.float32(2.0 * (F + 4.0) * U * (1.0 + F * 2.0**-21) * 1.0001))
    f_pad = (F + 31) // 32 * 32
    step = 64.0 * U * (f_pad // 16)
    e_rel = (2.0**-21 + step * (1 + 2.0**-10) + 4 * U) * (1 + 2.0**-10)
    kappa = (2 * e_rel + 2.5 * thr * (1 + (F + 2) * U)) / (1 - step) * (1 + 2.0**-10)
    return thr, kappa


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5, help="warm-up pairs")
    ap.add_argument("--launches", type=int, default=30, help="timed launches per schedule")
    args = ap.parse_args()

    import torch
    from ab_compact_rows import card

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
    routes = ("tc_bytes", "tc", "cuda_core")
    env = {"tc_bytes": {"UML_B200_LINEAR_TC": "1"},
           "tc": {"UML_B200_COMPACT_ROWS": "2", "UML_B200_LINEAR_TC": "1"},
           "cuda_core": {"UML_B200_LINEAR_TC": "0"}}
    labels = {r: torch.empty(n, dtype=torch.uint8, device="cuda") for r in routes}

    def step(route, want_stats=False):
        for k in ("UML_B200_COMPACT_ROWS", "UML_B200_LINEAR_TC"):
            os.environ.pop(k, None)
        os.environ.update(env[route])
        return eng.predict_peers(model, batch, [labels[route].data_ptr()], 0, exact=True, want_stats=want_stats,
                                 label_bytes=1)

    stats = {r: step(r, want_stats=True) for r in routes}
    os.environ["UML_B200_TC_REPLAY"] = "0"
    tier1 = {r: step(r, want_stats=True)["n_flagged"] for r in ("tc_bytes", "tc")}
    os.environ.pop("UML_B200_TC_REPLAY")
    assert [stats[r]["x_read_bytes"] for r in routes] == [1, 2, 2], stats
    equal = bool(torch.equal(labels["tc"], labels["cuda_core"]) and torch.equal(labels["tc_bytes"], labels["tc"]))
    before = card()
    for _ in range(args.warmup):
        for r in routes:
            step(r)
    ms = {r: [] for r in routes}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(args.launches):
        for r in routes:
            ev[0].record(stream)
            step(r)
            ev[1].record(stream)
            ev[1].synchronize()
            ms[r].append(ev[0].elapsed_time(ev[1]))
    after = card()
    for k in ("UML_B200_COMPACT_ROWS", "UML_B200_LINEAR_TC"):
        os.environ.pop(k, None)

    # float64 margins and A of every row, on the GPU in 1M-row chunks
    W = torch.tensor(np.asarray(arrs["coef"], dtype=np.float64), device="cuda")
    b = torch.tensor(np.asarray(arrs["intercept"], dtype=np.float64), device="cuda")
    wmax = W.abs().max(dim=0).values
    thr, kappa = thresholds(F)
    n_kappa = n_thr = 0
    for r0 in range(0, n, 1 << 20):
        x = torch.from_numpy(X[r0 : r0 + (1 << 20)]).to("cuda", torch.float64)
        top = torch.topk(x @ W.T + b, 2, dim=1).values
        m = top[:, 0] - top[:, 1]
        a = x.abs() @ wmax + b.abs().max()
        n_kappa += int((m <= kappa * a).sum())
        n_thr += int((m <= thr * a).sum())

    out = {"rows": n, "features": F, "launches_per_route": args.launches, "warmup_pairs": args.warmup,
           "labels_byte_equal": equal, "card_before": before, "card_after": after, "thr": thr, "kappa": kappa,
           "tier1_left_measured": tier1, "rows_margin_le_kappa_A": n_kappa, "rows_margin_le_thr_A": n_thr,
           "routes": {}}
    for r in routes:
        out["routes"][r] = {"ms_median": statistics.median(ms[r]), "ms_min": min(ms[r]), "ms_max": max(ms[r]),
                            "n_flagged": stats[r]["n_flagged"]}
    out["speedup_median"] = out["routes"]["cuda_core"]["ms_median"] / out["routes"]["tc"]["ms_median"]
    out["bytes_speedup_median"] = out["routes"]["tc"]["ms_median"] / out["routes"]["tc_bytes"]["ms_median"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
