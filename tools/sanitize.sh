#!/bin/sh
# Race / memory checking of the single-GPU kernels (SURVEY section 5 "race detection"): run on a GPU box, e.g.
#   sh tools/sanitize.sh > sanitize.log 2>&1
# memcheck: out-of-bounds / misaligned accesses; racecheck: shared-memory hazards (BN combine rows, stem, GEMM staging, resample bands).
set -x
K='bn_act_forward_backward and 256 or fused_sgd_flat_matches or normalize_kernel or metrics_kernel or multi_tensor_scale'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_kernels.py -q -x -k "$K" -p no:cacheprovider
echo "memcheck exit $?"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_stem.py -q -x -k "stem_forward_backward and dtype0 and shape0" -p no:cacheprovider
echo "racecheck(stem) exit $?"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_kernels.py -q -x -k "bn_act_forward_backward and 64 and dtype0" -p no:cacheprovider
echo "racecheck(bn) exit $?"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_tcgen05.py -q -x -k "shape0 or shape1" -p no:cacheprovider
echo "memcheck(gemm_bnstats) exit $?"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_fp64.py -q -x -k "one_cta_second_tile_n64" -p no:cacheprovider
echo "memcheck(gemm_bnstats, a CTA's second m-tile) exit $?"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_fp64.py -q -x -k "rpb3_odd_13x14_fp16_c32" -p no:cacheprovider
echo "racecheck(stem backward, quad rows crossing images) exit $?"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_fp16_gemm.py -q -x -k "geometry_edges and one_cta_second_tile_n64" -p no:cacheprovider
echo "memcheck(fp16 gemm_bnstats, a CTA's second m-tile) exit $?"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_fp16_gemm.py -q -x -k "stem_im2col and staged_224" -p no:cacheprovider
echo "racecheck(fp16 staged stem_im2col) exit $?"
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_data.py -q -x -k "equals_host_resample" -p no:cacheprovider
echo "memcheck(resample) exit $?"
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest "tests/test_gpu_data.py::test_device_resample_equals_host_resample[True]" -q -x -p no:cacheprovider
echo "racecheck(resample bands) exit $?"
