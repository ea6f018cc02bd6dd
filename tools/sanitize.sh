# compute-sanitizer over tools/sanitize_target.py (final default kernels: item / packet / spread / batch / shard / peer-flag paths,
# and every entry point that writes device memory, at the small sizes of tests/test_memory_contract.py).
# Writes gpurun_out/r2_sanitizer_<tool>.txt; copy the summaries into profiles/.
set -x
for tool in memcheck initcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 python tools/sanitize_target.py > gpurun_out/r2_sanitizer_$tool.txt 2>&1
  echo "$tool rc=$?"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|SANITIZE_TARGET|hazard" gpurun_out/r2_sanitizer_$tool.txt | tail -n 5
done
