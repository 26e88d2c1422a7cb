#!/bin/bash
# Read ceiling + feed-only + wait-clock + timeline breakdown of the linear tile kernel (tools/linear_probe.cu), on GPU 0,
# for each schedule: chunked and whole fp32 rows, and the compact fp16 rows (whose feed-only and wait-clock lines say
# whether that schedule is bound by its feed or by its scoring warps), and the feed of the byte rows' 16 KiB stages
# against the read ceiling over their 0.64 GB; then the fp16 schedule without its W loads,
# without its x loads, and with neither; then the fp16 schedule with 4 rows per lane per pass and with the library's 8,
# alternating (both with four scoring warps and 256-row stages); then the byte schedule without its per-row epilogue
# (its epilogue warps hand every score slot back unread) and without its queue hand-off.
# Writes MEASURED_PEAKS.json (the read ceiling bench.py's roofline divides by) and the probe's JSON lines to
# ${1:-build/probe}/linear_probe.jsonl.  Binaries go to build/probe/.
set -euo pipefail
cd "$(dirname "$0")/.."
out=${1:-build/probe}
mkdir -p build/probe "$out"
nvcc=${NVCC:-$(command -v nvcc || echo /usr/local/cuda/bin/nvcc)}
flags=(-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -DUML_PROBE_CLASSES=10)
declare -A defs=([plain]="" [feed_only]="-DUML_PROBE_FEED_ONLY" [wait_clocks]="-DUML_PROBE_WAIT_CLOCKS" [timeline]="-DUML_PROBE_TIMELINE"
                 [no_w_loads]="-DUML_PROBE_NO_W" [no_x_loads]="-DUML_PROBE_NO_X" [math_only]="-DUML_PROBE_NO_W -DUML_PROBE_NO_X"
                 [half_only]="-DUML_PROBE_HALF_ONLY" [half_only_rows4]="-DUML_PROBE_HALF_ONLY -DUML_PROBE_HALF_PASS_ROWS=4"
                 [no_epilogue]="-DUML_PROBE_NO_EPILOGUE" [no_handoff]="-DUML_PROBE_NO_HANDOFF")
variants=(plain feed_only wait_clocks timeline no_w_loads no_x_loads math_only half_only_rows4 half_only no_epilogue no_handoff)
for v in "${variants[@]}"; do
  bin=build/probe/linear_probe_$v
  if [ ! -x "$bin" ] || [ tools/linear_probe.cu -nt "$bin" ] || [ unionml_b200/csrc/linear_kernels.cu -nt "$bin" ] ||
     [ unionml_b200/csrc/linear_tc_kernels.cu -nt "$bin" ] || [ unionml_b200/csrc/linear_tile.cuh -nt "$bin" ] ||
     [ unionml_b200/csrc/uml_common.cuh -nt "$bin" ] || [ unionml_b200/csrc/label_store.cuh -nt "$bin" ]; then
    "$nvcc" "${flags[@]}" ${defs[$v]} tools/linear_probe.cu -o "$bin" &
  fi
done
wait
nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader | sed 's/^/# before: /' | tee -a "$out/linear_probe.jsonl"
for v in "${variants[@]}" half_only_rows4 half_only; do
  build/probe/linear_probe_$v | tee -a "$out/linear_probe.jsonl"
done
nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader | sed 's/^/# after: /' | tee -a "$out/linear_probe.jsonl"
python3 - "$out/linear_probe.jsonl" <<'PY'
import json, sys
rows = [json.loads(l) for l in open(sys.argv[1]) if l.startswith("{")]
ceiling = [r for r in rows if r["probe"] == "read_ceiling"][-1]  # the 2.56 GB one (fp32 rows of the cfg2 shape)
json.dump({"hbm_gbs": ceiling["hbm_gbs"], "device": ceiling["device"],
           "method": "tools/linear_probe.cu read_kernel, 2.56 GB, 16-byte ld.global.nc.L1::no_allocate, >= 0.5 s"},
          open("MEASURED_PEAKS.json", "w"))
print("MEASURED_PEAKS.json:", ceiling["hbm_gbs"], "GB/s")
PY
