#!/bin/bash
# compute-sanitizer over the hot path (SURVEY.md section 5: race detection / sanitizers hook).
#   memcheck  : out-of-bounds / misaligned global and shared accesses, leaks of device memory
#   racecheck : shared-memory hazards (k_linear_memories_band staging, k_coarse_packed task queue + bit-planes,
#               k_refine<true> / k_refine_bits partial sums, block scans)
#   synccheck : barrier / mbarrier misuse (the TMA staging of k_coarse_packed, __syncthreads in divergent code)
# on (a) __graft_entry__.smoke() -- one full match checked against the oracle -- and (b) the fused multi-GPU exchange
# with three handles in one process (peer stores, ticket counters, frame flags, the collector's spin wait), and
# (c) memcheck over the frames and banks that route the refinement to its byte-wise kernels: k_refine<false> on frames
# the filter does not take, k_refine<true> behind the filter (unsafe templates, three levels), k_refine_prep deriving the
# H-planes from the byte linear memories, and (d) memcheck over lm_detect_batch: a batch whose survivors span two pose
# chunks, and one with early returns and NaN anchors, and (e) the pose stage shared over two handles of one process (peer
# stores of the ICP kernel, its ticket and pose flags, the pose collector's spin wait), and (f) memcheck over
# lm_peer_detect_batch with three handles of one process: a shared batch of two pose chunks, one with fewer survivors
# than ranks and an all-blank one (k_pose_cloud's slot and frame indexing of a shared chunk, the per-chunk pose exchanges).
# Usage (on a GPU box):  bash tools/sanitize.sh [outdir]      -> <outdir>/summary.txt, one log per tool x case
set -u
OUT=${1:-gpurun_out/sanitize}
mkdir -p "$OUT"
export LINEMOD_B200_PEER_TIMEOUT_MS=600000   # kernels run 10-100x slower under the sanitizer: no false peer timeouts
CS=${CS:-compute-sanitizer}
: > "$OUT/summary.txt"
run() {  # tool case command...
  local tool=$1 name=$2; shift 2
  local log="$OUT/${tool}_${name}.log"
  local extra=""
  [ "${CS_LEAK:-0}" = 1 ] && extra="--leak-check full"
  timeout 900 $CS --tool "$tool" $extra --error-exitcode 7 --print-limit 20 --log-file "$log" "$@" > "$OUT/${tool}_${name}.out" 2>&1
  local rc=$?
  local errs
  errs=$(grep -E "ERROR SUMMARY|RACECHECK SUMMARY" "$log" | tail -1)
  local leaks
  leaks=$(grep -E "LEAK SUMMARY" "$log" | tail -1)
  echo "$tool $name rc=$rc :: ${errs:-no summary line}${leaks:+ $leaks}" | tee -a "$OUT/summary.txt"
}
for tool in memcheck racecheck synccheck; do
  run "$tool" smoke python -c "import __graft_entry__ as g; g.smoke()"
  run "$tool" exchange3 python -m pytest "tests/test_gpu_dist.py::test_fused_exchange_three_handles_one_process" -x -q -p no:cacheprovider
done
run memcheck refine_routes python -m pytest "tests/test_gpu_refine_bounds.py::test_zero_score_patches" \
  "tests/test_gpu_match_parity.py::test_match_bit_exact_synthetic[T6-640-512-96-35-70.0]" -x -q -p no:cacheprovider
run memcheck detect_batch python -m pytest "tests/test_gpu_detect_batch.py::test_survivors_beyond_one_chunk" \
  "tests/test_gpu_detect_batch.py::test_early_returns_and_nan_anchors" -x -q -p no:cacheprovider
for tool in memcheck racecheck synccheck; do
  run "$tool" pose_share2 python -m pytest "tests/test_gpu_pose_share.py::test_every_rank_returns_the_single_gpu_result[2]" -x -q \
    -p no:cacheprovider
done
run memcheck peer_batch3 python -m pytest "tests/test_gpu_peer_batch.py::test_two_chunks_few_survivors_and_a_blank_batch" -x -q \
  -p no:cacheprovider
# (g) leaks: a detector's batch with pose stage, pose NMS and timing, and one ICP call, both handles closed explicitly;
# the summary must list no leaked allocation (every buffer the handles own is freed with them)
CS_LEAK=1 run memcheck leaks python tools/leak_probe.py
echo "done: $(cat "$OUT/summary.txt" | wc -l) runs" | tee -a "$OUT/summary.txt"
