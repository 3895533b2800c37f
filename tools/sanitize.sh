#!/usr/bin/env bash
# compute-sanitizer over the smoke path (SURVEY.md §5 "race detection"): memcheck finds out-of-bounds / misaligned accesses
# of the hand-written kernels, racecheck shared-memory hazards, synccheck barrier misuse.  On a machine with a GPU and
# compute-sanitizer:
#     bash tools/sanitize.sh memcheck > sanitize_memcheck.log 2>&1
# The TMA / wgmma kernels are covered by memcheck (global side) only: racecheck does not model the async proxy.
set -u
TOOL=${1:-memcheck}
cd "$(dirname "$0")/.."
exec timeout 1400 compute-sanitizer --tool "$TOOL" --error-exitcode 7 --launch-timeout 120 \
    python -c "import __graft_entry__ as g; g.smoke()"
