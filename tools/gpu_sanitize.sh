#!/bin/bash
# compute-sanitizer over the walk kernel that SHIPS for the headline geometry (D = 12, F = 256, AUTO plan =
# dt_walk_tile<4,2,1,0,384>, phased ring refill, CTAs with two tiles) and over the planner's alternatives.
# Logs (with the kernel name printed by the test) go to <logdir>/sanitizer_<tool>_<plan>.log.
#   bash tools/gpu_sanitize.sh [logdir=sanitizer_logs]   memcheck + synccheck over six launch plans (two of them
#                                                        with split tree tops, DTE_TUNE tops=6), a 3-class
#                                                        ensemble, seven kernel-matrix instantiations, the binned and
#                                                        the leaf walks, memcheck over the sparse densify kernel,
#                                                        leak checks of the C++ host on a three-position ring,
#                                                        racecheck
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
  # split tree tops (dt_walk_tile_split): the two-stage plan the cfg3 handle measures fastest, and a phased one
  for tune in "pair=4,stages=2,phased=0,tops=6" "pair=4,stages=1,phased=1,tops=6"; do run $tool "$tune" ""; done
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
# the sparse densify kernel (sparse_rows_kernel): rows with duplicates, skipped indices and indptr[0] != 0, on its own
# and in front of the walk, host and device
for T in tests/test_gpu_sparse.py::test_sparse_to_dense_device_bytes "tests/test_gpu_sparse.py::test_host_counts_pinned_pageable_scipy[5003]" \
         tests/test_gpu_sparse.py::test_device_side_stream_and_chunks; do
  stag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  run memcheck "" ""; mv "$OUT/sanitizer_memcheck_auto.log" "$OUT/sanitizer_memcheck_sparse_${stag}.log"
done
# the contribution kernels (dt_shap_tile with two tuple groups per CTA, dt_shap_generic at a width only it serves and in
# two launches through its fp64 scratch), the ragged tail of a warp, and both <15> kernels on D = 15 paths of 15 elements
# with the bottom-up unwinding (covers above their parent's)
for T in tests/test_gpu_contribs.py::test_headline_geometry tests/test_gpu_contribs.py::test_generic_only_width \
         tests/test_gpu_contribs.py::test_generic_launches_in_chunks "tests/test_gpu_contribs.py::test_tuple_counts[33]" \
         "tests/test_gpu_contribs_deep.py::test_leafwise_merged_lengths[m15-D15-free]"; do
  ctag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  run memcheck "" ""; mv "$OUT/sanitizer_memcheck_auto.log" "$OUT/sanitizer_memcheck_contribs_${ctag}.log"
done
# the interaction kernel: several row blocks through the fp64 scratch, three launch chunks, the ragged tail of a warp and
# the <15> kernel on D = 15 paths with the bottom-up unwinding
for T in tests/test_gpu_interactions.py::test_row_blocks_give_the_same_bytes tests/test_gpu_interactions.py::test_several_launch_chunks \
         "tests/test_gpu_interactions.py::test_tuple_counts[33]" "tests/test_gpu_interactions.py::test_deep_leafwise[free-15-15-15]"; do
  itag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  run memcheck "" ""; mv "$OUT/sanitizer_memcheck_auto.log" "$OUT/sanitizer_memcheck_inter_${itag}.log"
done
# the approximate contributions: both passes (the leaf walk into the cell scratch, dt_approx_generic from it) at D = 15,
# at F = 2048, in two scratch chunks, on the ragged tail of a warp, and with three classes on a tree chunk
for T in "tests/test_gpu_approx_contribs.py::test_depths_and_widths[D15-F4]" "tests/test_gpu_approx_contribs.py::test_depths_and_widths[D3-F2048]" \
         tests/test_gpu_approx_contribs.py::test_two_scratch_chunks "tests/test_gpu_approx_contribs.py::test_tuple_counts[33]" \
         tests/test_gpu_approx_contribs.py::test_classes_and_a_chunk; do
  atag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  run memcheck "" ""; mv "$OUT/sanitizer_memcheck_auto.log" "$OUT/sanitizer_memcheck_approx_${atag}.log"
done
# the interventional kernel: the <3>, <7> and <15> instantiations on leaf-wise deep trees, a ragged block of 32 background
# rows and 1000 rows, two launches through the fp64 scratch at F = 2048, the ragged tail of a warp and three classes on a
# tree chunk; synccheck and racecheck over the shared-memory G table its blocks fill before the __syncthreads
for T in "tests/test_gpu_interventional.py::test_leafwise_bounds[D13-M3]" "tests/test_gpu_interventional.py::test_leafwise_bounds[D14-M7]" \
         "tests/test_gpu_interventional.py::test_leafwise_bounds[D15-M15]" \
         "tests/test_gpu_interventional.py::test_background_sizes[33]" "tests/test_gpu_interventional.py::test_background_sizes[1000]" \
         tests/test_gpu_interventional.py::test_several_scratch_launches "tests/test_gpu_interventional.py::test_tuple_counts[33]" \
         tests/test_gpu_interventional.py::test_classes_and_a_chunk; do
  vtag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  run memcheck "" ""; mv "$OUT/sanitizer_memcheck_auto.log" "$OUT/sanitizer_memcheck_interv_${vtag}.log"
done
T="tests/test_gpu_interventional.py::test_background_sizes[33]"
run synccheck "" ""; mv "$OUT/sanitizer_synccheck_auto.log" "$OUT/sanitizer_synccheck_interv.log"
run racecheck "" "--racecheck-report all"; mv "$OUT/sanitizer_racecheck_auto.log" "$OUT/sanitizer_racecheck_interv.log"
# the categorical walks: dt_walk_tile_cat and dt_walk_generic_cat, single-class and three classes, at D = 1 and D = 15,
# at the tile's widest F and at F = 2048, and on the ragged tail of a warp
for T in "tests/test_gpu_categorical.py::test_bit_exact_against_the_expansion[1-16-8-1-1-1-33]" \
         "tests/test_gpu_categorical.py::test_bit_exact_against_the_expansion[15-8-16-1-1-1-200]" \
         "tests/test_gpu_categorical.py::test_bit_exact_against_the_expansion[3-30-8-2-2-3-33]" \
         "tests/test_gpu_categorical.py::test_bit_exact_against_the_expansion[15-6-8-1-1-3-64]" \
         "tests/test_gpu_categorical.py::test_tile_generic_boundary_and_widest_tuples[1816]" \
         "tests/test_gpu_categorical.py::test_tile_generic_boundary_and_widest_tuples[2048]" \
         tests/test_gpu_categorical.py::test_kats_on_the_device; do
  ctag=$(echo "${T##*::}" | tr -c 'A-Za-z0-9\n' '_')
  run memcheck "" ""; mv "$OUT/sanitizer_memcheck_auto.log" "$OUT/sanitizer_memcheck_cat_${ctag}.log"
done
# leaks: the C++ host (no torch caching allocator in the process) over a handle's whole life, create to destroy, on three
# ring positions sharing one GPU, data- and ensemble-sharded, fed by the line stream and by the host fast path
for mode in stream host; do
  for part in data ensemble; do
    log=$OUT/sanitizer_memcheck_leaks_${mode}_${part}.log
    timeout 900 compute-sanitizer --tool memcheck --leak-check full --error-exitcode 7 tools/dte_host 48 6 256 6000 4 $mode 0,0,0 $part > "$log" 2>&1
    echo "memcheck leaks [$mode $part] rc=$? $(grep -E 'ERROR SUMMARY|LEAK SUMMARY|leaked' "$log" | tr '\n' ' ' | cut -c1-300)"
  done
done
T=tests/test_gpu_parity.py::test_shipped_plan_headline_geometry_multi_tile
timeout 300 compute-sanitizer --tool racecheck --racecheck-report all --print-limit 8 --show-backtrace no tools/racecheck_canonical > $OUT/sanitizer_racecheck_canonical.log 2>&1
echo "racecheck [canonical textbook pipeline] rc=$? $(grep -E 'canonical|RACECHECK SUMMARY' $OUT/sanitizer_racecheck_canonical.log | tr '\n' ' ' | cut -c1-300)"
run racecheck "" "--racecheck-report all"
