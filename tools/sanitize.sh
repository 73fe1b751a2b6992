#!/bin/bash
# compute-sanitizer over the smoke shapes of every hand-synchronised kernel (run on a machine with a GPU: bash tools/sanitize.sh).
# memcheck: out-of-bounds / misaligned accesses incl. shared memory and TMA destinations; racecheck: shared-memory hazards between
# the gather warps, the epilogue and the A/B panel writers.
cd "$(dirname "$0")/.."
out="${TMPDIR:-/tmp}/stmp_sanitizer"; mkdir -p "$out"
for tool in memcheck racecheck; do
  timeout 330 compute-sanitizer --tool $tool --print-limit 30 python tools/sanitize_smoke.py > "$out/$tool.txt" 2>&1
  echo "[$tool] rc=$?" >> "$out/$tool.txt"
  tail -4 "$out/$tool.txt"
done
