#!/bin/bash
# compute-sanitizer passes over small shapes (SURVEY.md section 4 item 4).  Run on a GPU box:
#   gpurun --timeout 2400 -- tools/sanitize.sh
# memcheck: the paths written in round 2 (gathered column direction, sharded upload, warp 5-point solver, batched
# estimator, distortion models); racecheck / synccheck: the K1 GEMM kernel (cluster-scope mbarrier protocol), the gather
# and resolve kernels and the RANSAC kernels on tiny inputs.  Logs go to gpurun_out/ (copy the ones to keep to profiles/).
set -u
mkdir -p gpurun_out
S=/usr/local/cuda/bin/compute-sanitizer
T="timeout 900"
$T $S --tool memcheck --error-exitcode 1 python -m pytest -q -x -m gpu -p no:cacheprovider tests/test_zz_native_gpu.py \
    -k "column_direction_skip or sharded or five_point or batched_two_view or distortion_oracle" > gpurun_out/sanitize_memcheck.log 2>&1
echo "memcheck exit $?" | tee -a gpurun_out/sanitize_memcheck.log
# guided matching (split residual, gathered column direction), the overlapped order and the warp eigen-solve of the LO refits
$T $S --tool memcheck --error-exitcode 1 python -m pytest -q -x -m gpu -p no:cacheprovider tests/test_verify_gpu.py tests/test_zz_native_gpu.py \
    -k "guided_matching_h_kind or warp_eigen or overlapped_schedule" > gpurun_out/sanitize_memcheck_r2late.log 2>&1
echo "memcheck (guided / overlap / eigen) exit $?" | tee -a gpurun_out/sanitize_memcheck_r2late.log
$T $S --tool racecheck --error-exitcode 1 python -m pytest -q -x -m gpu -p no:cacheprovider tests/test_match_gpu.py -k "identity_and_reverse or empty_inputs or ties_zeros" \
    > gpurun_out/sanitize_racecheck.log 2>&1
echo "racecheck exit $?" | tee -a gpurun_out/sanitize_racecheck.log
$T $S --tool synccheck --error-exitcode 1 python -m pytest -q -x -m gpu -p no:cacheprovider tests/test_match_gpu.py -k "identity_and_reverse" \
    > gpurun_out/sanitize_synccheck.log 2>&1
echo "synccheck exit $?" | tee -a gpurun_out/sanitize_synccheck.log
DIAG_N=120 DIAG_REPS=1 $T $S --tool racecheck --error-exitcode 1 python tools/diag_determinism.py > gpurun_out/sanitize_racecheck_verifier.log 2>&1
echo "racecheck (verifier) exit $?" | tee -a gpurun_out/sanitize_racecheck_verifier.log
# absolute pose: the RANSAC, selection and refinement kernels on small shapes (logs under $ABS_LOGS, default out/)
ABS_LOGS=${ABS_LOGS:-out}
mkdir -p "$ABS_LOGS"
$T $S --tool memcheck --error-exitcode 1 python -m pytest -q -x -m gpu -p no:cacheprovider tests/test_zz_abs_pose_gpu.py \
    -k "not 4097" > $ABS_LOGS/sanitize_memcheck_abs_pose.log 2>&1
echo "memcheck (absolute pose) exit $?" | tee -a $ABS_LOGS/sanitize_memcheck_abs_pose.log
$T $S --tool racecheck --error-exitcode 1 python -m pytest -q -x -m gpu -p no:cacheprovider tests/test_zz_abs_pose_gpu.py \
    -k "covariance or pose_refinement" > $ABS_LOGS/sanitize_racecheck_abs_pose.log 2>&1
echo "racecheck (absolute pose) exit $?" | tee -a $ABS_LOGS/sanitize_racecheck_abs_pose.log
tail -n 4 gpurun_out/sanitize_*.log
tail -n 4 "$ABS_LOGS"/sanitize_*_abs_pose.log
