#!/bin/bash
# compute-sanitizer passes over the shipped kernels at small sizes (summary lines -> gpurun_out/sanitizer.txt)
# (the fourth pass, memcheck under UML_B200_RESCORE_MODE=kernel, covers the linear re-score kernel behind small models)
passes() {
for tool in "$@"; do
  echo "== compute-sanitizer --tool $tool python tools/sanitize_driver.py" >> gpurun_out/sanitizer.txt
  timeout 280 compute-sanitizer --tool $tool python tools/sanitize_driver.py 2>&1 | grep -E "sanitizer driver ok|ERROR SUMMARY|RACECHECK SUMMARY|Error|hazard" | head -12 >> gpurun_out/sanitizer.txt
done
}
passes memcheck racecheck synccheck
UML_B200_RESCORE_MODE=kernel passes memcheck
