"""Same-box A/B runs (box-to-box variation on this pool is ~10 %, so only same-call comparisons count):
  * linear step: default (flag list + PDL-launched re-score kernel) vs re-score inside the tile kernel
    (UML_B200_RESCORE_MODE=queue: shared-memory queue + re-score warp) vs plain launches (UML_B200_NO_PDL=1), 10M and 1.25M rows
  * MLP step: tensor-core kernel vs CUDA-core kernel (UML_B200_MLP_TC=0)
Each variant runs in its own process (the switches are read once).  Prints one JSON object."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
WORKER = r'''
import json, sys, numpy as np, torch
sys.path.insert(0, %r)
from unionml_b200.engine import Engine
what, rows = sys.argv[1], int(sys.argv[2])
F = int(sys.argv[3]) if len(sys.argv) > 3 else 64
dev = torch.device("cuda", 0); eng = Engine(0)
s = torch.cuda.Stream(device=dev); torch.cuda.set_stream(s); eng.set_stream(s.cuda_stream)
X = torch.randint(0, 17, (rows, F), device=dev, dtype=torch.int32).to(torch.float32) if F == 64 else torch.randint(0, 256, (rows, F), device=dev, dtype=torch.int32).to(torch.float32) / 255.0
b = eng.wrap_device(X.data_ptr(), rows, F, keepalive=X)
lab = torch.empty(rows, dtype=torch.uint8, device=dev)
if what == "linear":
    z = np.load(%r)
    m = eng.load_linear(z["coef"], z["intercept"]) if F == 64 else eng.load_linear((np.random.default_rng(1).standard_normal((10, F)) * 0.05).astype(np.float32), np.random.default_rng(2).standard_normal(10).astype(np.float32))
    run = lambda st=False: eng.predict_peers(m, b, [lab.data_ptr()], 0, exact=True, want_stats=st, label_bytes=1)
else:
    z = np.load(%r); m = eng.load_mlp(z["w1"], z["b1"], z["w2"], z["b2"])
    run = lambda st=False: eng.predict_mlp_peers(m, b, [lab.data_ptr()], 0, exact=True, want_stats=st, label_bytes=1)
for _ in range(10): run()
torch.cuda.synchronize()
best = 1e9
for rep in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(40): run()
    e1.record(s); torch.cuda.synchronize()
    best = min(best, e0.elapsed_time(e1) / 40)
st = run(True)
print(json.dumps({"ms_per_step": best, "kernel_ms": st["kernel_ms"], "recheck_ms": st["recheck_ms"], "flagged": st["n_flagged"],
                  "launches": st["kernel_launches"], "path": st["path"], "checksum": int(lab.to(torch.int64).sum().item())}))
''' % (str(ROOT), str(ROOT / "tests/golden/digits_lr.npz"), str(ROOT / "tests/golden/mlp_64_32_10.npz"))


def run(what, rows, env, F=64):
    r = subprocess.run([sys.executable, "-c", WORKER, what, str(rows), str(F)], env=dict(os.environ, **env), capture_output=True, text=True, timeout=300)
    if r.returncode != 0:
        return {"error": r.stderr[-600:]}
    return json.loads(r.stdout.strip().splitlines()[-1])


out = {}
for rows in (10_000_000, 1_250_000):
    out[f"linear_{rows}"] = {"default": run("linear", rows, {}), "rescore_kernel": run("linear", rows, {"UML_B200_RESCORE_MODE": "kernel"}),
                             "no_pdl": run("linear", rows, {"UML_B200_NO_PDL": "1"}), "default_again": run("linear", rows, {})}
out["linear_784_2000000"] = {"default": run("linear", 2_000_000, {}, 784), "rescore_kernel": run("linear", 2_000_000, {"UML_B200_RESCORE_MODE": "kernel"}, 784)}
out["mlp_10000000"] = {"tc": run("mlp", 10_000_000, {}), "ffma": run("mlp", 10_000_000, {"UML_B200_MLP_TC": "0"})}
out["mlp_1250000"] = {"tc": run("mlp", 1_250_000, {}), "ffma": run("mlp", 1_250_000, {"UML_B200_MLP_TC": "0"})}
print(json.dumps(out, indent=1))
