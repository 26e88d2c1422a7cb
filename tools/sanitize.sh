#!/bin/bash
# compute-sanitizer passes over the shipped kernels at small sizes (summary lines -> gpurun_out/sanitizer.txt)
# (UML_B200_MLP_RESCORE_MODE=queue is exercised in a second memcheck pass: the in-kernel re-score warps of the tensor-core kernel)
for tool in memcheck racecheck synccheck; do
  echo "== compute-sanitizer --tool $tool python tools/sanitize_driver.py" >> gpurun_out/sanitizer.txt
  timeout 280 compute-sanitizer --tool $tool python tools/sanitize_driver.py 2>&1 | grep -E "sanitizer driver ok|ERROR SUMMARY|RACECHECK SUMMARY|Error|hazard" | head -12 >> gpurun_out/sanitizer.txt
done
echo "== UML_B200_MLP_RESCORE_MODE=queue UML_B200_RESCORE_MODE=kernel compute-sanitizer --tool memcheck python tools/sanitize_driver.py" >> gpurun_out/sanitizer.txt
UML_B200_MLP_RESCORE_MODE=queue UML_B200_RESCORE_MODE=kernel timeout 280 compute-sanitizer --tool memcheck python tools/sanitize_driver.py 2>&1 | grep -E "sanitizer driver ok|ERROR SUMMARY|Error" | head -12 >> gpurun_out/sanitizer.txt
