#!/bin/bash
# Race / memory / sync checking of the native engine under compute-sanitizer (run on a GPU machine where
# compute-sanitizer works: `bash scripts/sanitize.sh`).  The reference has no sanitizer story at all (SURVEY.md section 5);
# here the engine has real concurrency (streams, TMA/async proxy, peer-memory flags), so these are the
# three standard passes.  Eager mode (--no-graph) so every launch is attributed; tiny step counts because
# the tools slow kernels down by 10-100x (the device-side spin limit is 4 s).
set -u
ARGS="bench.py --steps 2 --warmup 3 --repeats 1 --no-alt --no-graph --pool-batches 4"
for tool in memcheck racecheck synccheck; do
    echo "== compute-sanitizer --tool $tool"
    timeout 900 compute-sanitizer --tool $tool --print-limit 5 python $ARGS 2>&1 | grep -E "Error: |ERROR SUMMARY|RACECHECK SUMMARY" | cut -c1-260 | head -12
done
# SSB_RACECHECK=1 adds one more named barrier per layer among the chain kernel's math warps around the reuse of its
# activation ping-pong tiles; the run must be clean with and without it.
echo "== compute-sanitizer --tool racecheck, SSB_RACECHECK=1 (extra per-layer barrier among the math warps)"
SSB_RACECHECK=1 timeout 900 compute-sanitizer --tool racecheck --print-limit 5 python $ARGS 2>&1 | grep -E "Error: |ERROR SUMMARY|RACECHECK SUMMARY" | cut -c1-260 | head -12
echo "== serialized-streams debug mode (SSB_SERIALIZE=1): results must not change"
SSB_SERIALIZE=1 timeout 300 python bench.py --steps 20 --warmup 3 --no-graph 2>&1 | grep "^{" | cut -c1-160
