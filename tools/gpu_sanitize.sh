#!/bin/bash
# compute-sanitizer over the walk kernel that SHIPS for the headline geometry (D = 12, F = 256, AUTO plan =
# dt_walk_tile<4,2,1,0,384>, phased ring refill, CTAs with two tiles) and over the planner's alternatives.
# Logs (with the kernel name printed by the test) go to <logdir>/sanitizer_<tool>_<plan>.log.
#   bash tools/gpu_sanitize.sh [logdir=sanitizer_logs]   memcheck + synccheck over four launch plans, a 3-class
#                                                        ensemble, seven kernel-matrix instantiations, the binned and
#                                                        the leaf walks, racecheck
#                                                        once (AUTO)
# racecheck does not model the mbarrier / cp.async.bulk (async-proxy) hand-off: tools/racecheck_canonical.cu is the
# textbook producer/consumer ring with exactly that synchronisation, run under the same tool for comparison.
set -u
OUT=${1:-sanitizer_logs}
mkdir -p "$OUT"
export DTE_TEST_SANITIZER=1
T=tests/test_gpu_parity.py::test_shipped_plan_headline_geometry_multi_tile
run() { # tool tune extra-args
  tag=$(echo "${2:-auto}" | tr ',=' '__')
  log=$OUT/sanitizer_$1_${tag}.log
  DTE_TUNE="$2" timeout 900 compute-sanitizer --tool $1 $3 --error-exitcode 7 --print-limit 8 --show-backtrace no \
      python -m pytest "$T" -q -x -s > "$log" 2>&1
  echo "$1 [$tag] rc=$? $(grep -E 'shipped-plan|ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' "$log" | tr '\n' ' ' | cut -c1-400)"
}
for tool in memcheck synccheck; do
  for tune in "" "pair=4,stages=1" "pair=1,ilp=8,stages=1" "pair=2,ilp=2,stages=2"; do run $tool "$tune" ""; done
done
# the multi-class epilogue (C = 3, class-boundary stores and the argmax read-back) in the same geometry
T=tests/test_gpu_multiclass.py::test_multiclass_headline_geometry_multi_tile
for tool in memcheck synccheck; do run $tool "" "" ; mv "$OUT/sanitizer_${tool}_auto.log" "$OUT/sanitizer_${tool}_multiclass.log"; done
# instantiations no other test launches, from the kernel matrix (each case pins its own DTE_TUNE; one wave of CTAs
# + 33 tuples here): the wide-record staged kernels but <4,2,1,1,384>, the P = 4 compact <2,4,1,0,384> and the
# non-staged wide <4,1,0,1,384>
for id in "dt_walk_tile<8,1,1,1,288>-C1-typical-D10-F516" "dt_walk_tile<4,1,1,1,384>-C1-typical-D10-F516" \
          "dt_walk_tile<2,2,1,1,384>-C1-typical-D10-F516" "dt_walk_tile<2,4,1,1,384>-C1-typical-D10-F516" \
          "dt_walk_tile<2,4,1,1,672>-C1-typical-D10-F516" "dt_walk_tile<2,4,1,0,384>-C1-typical-D11-F512" \
          "dt_walk_tile<4,1,0,1,384>-C1-typical-D10-F516"; do
  T="tests/test_gpu_kernel_matrix.py::test_reachable_instantiation_bit_exact[$id]"
  ktag=$(echo "$id" | cut -d- -f1 | tr -c 'A-Za-z0-9\n' '_')      # run() sets its own $tag
  for tool in memcheck synccheck; do run $tool "" ""; mv "$OUT/sanitizer_${tool}_auto.log" "$OUT/sanitizer_${tool}_matrix_${ktag}.log"; done
done
# the binned walk (u8 tile, 4-byte tops): the headline plan (phased), the D = 5 staged plan that must not phase, and a
# non-staged plan (D = 3 has one top level and is never staged)
for T in tests/test_gpu_binned.py::test_headline_binned_multi_tile tests/test_gpu_binned.py::test_phased_at_depth_5_stays_unphased \
         "tests/test_gpu_binned.py::test_depths[3]"; do
  btag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  for tool in memcheck synccheck; do run $tool "" ""; mv "$OUT/sanitizer_${tool}_auto.log" "$OUT/sanitizer_${tool}_binned_${btag}.log"; done
done
# the leaf walk (cell stores instead of the reduction): the headline plan with three tiles per CTA, and the generic kernel
for T in tests/test_gpu_leaves.py::test_headline_leaf_plan_multi_tile "tests/test_gpu_leaves.py::test_small_batches[33]"; do
  ltag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  for tool in memcheck synccheck; do run $tool "" ""; mv "$OUT/sanitizer_${tool}_auto.log" "$OUT/sanitizer_${tool}_leaf_${ltag}.log"; done
done
T=tests/test_gpu_parity.py::test_shipped_plan_headline_geometry_multi_tile
timeout 300 compute-sanitizer --tool racecheck --racecheck-report all --print-limit 8 --show-backtrace no tools/racecheck_canonical > $OUT/sanitizer_racecheck_canonical.log 2>&1
echo "racecheck [canonical textbook pipeline] rc=$? $(grep -E 'canonical|RACECHECK SUMMARY' $OUT/sanitizer_racecheck_canonical.log | tr '\n' ' ' | cut -c1-300)"
run racecheck "" "--racecheck-report all"
