#!/usr/bin/env bash
# compute-sanitizer passes over the kernel numerics tests at CI-sized shapes (SURVEY §5.2): fused ops, GEMM (bf16 + fp8), the fp8
# producers, attention fwd/bwd, and the NVLink kernels (fed_round / ddp_allreduce / ddp_zero_step run on one GPU with n = 1, plus the
# single-process multi-GPU tests when the box has peers).
# usage (on a GPU box): scripts/sanitize.sh [memcheck|racecheck|synccheck|initcheck|all]
set -uo pipefail
cd "$(dirname "${BASH_SOURCE[0]}")/.."; mkdir -p gpurun_out
TOOLS=${1:-memcheck}
[ "$TOOLS" = all ] && TOOLS="memcheck racecheck synccheck initcheck"
SEL='layernorm or cross_entropy or embedding or colsum or optimizer or gemm_kk_bias or gemm_fp8_forward or gemm_fp8_wgrad or gelu_epilogue or weight_segments or test_attention_fwd or test_attention_bwd or fed_round_matches_oracle or allreduce'
# synccheck treats an mbarrier phase that completes without a waiter as "Missing wait" and kills the kernel: the attention kernels
# commit `pv_done` after every P·V but only wait on it when a row's reference maximum moved (a rescale) — by design — so they are
# left out of the synccheck pass; initcheck tracks every global byte and is run on a smaller selection. memcheck also covers the
# scoring kernels (cache attention, slotted cache append), the embedding backward without a token-embedding gradient and the
# ZeRO-3 E4M3 requantisation kernel at world size 1.
rc=0
for TOOL in $TOOLS; do
  CUR="$SEL"
  EXTRA=""
  [ "$TOOL" = memcheck ] && CUR="$SEL or cache_attention or slotted_decode_append or embed_bwd_without or requant_kernel" \
    && EXTRA="tests/test_frozen_gpu.py tests/test_zero3_fp8_gpu.py"
  [ "$TOOL" = synccheck ] && CUR="layernorm or cross_entropy or embedding or colsum or optimizer or gemm_kk_bias or gemm_fp8_forward or gemm_fp8_wgrad or gelu_epilogue or weight_segments or fed_round_matches_oracle or allreduce"
  [ "$TOOL" = initcheck ] && CUR="layernorm or gemm_kk_bias or gemm_fp8_wgrad or weight_segments or (fed_round_matches_oracle and fedadam)"
  compute-sanitizer --tool "$TOOL" --error-exitcode 3 --print-limit 20 \
    python -m pytest tests/test_kernels_gpu.py tests/test_fp8_gpu.py tests/test_attention_gpu.py tests/test_score_gpu.py tests/test_multigpu.py $EXTRA -x -q -k "$CUR" \
    2>&1 | tail -25 | tee "gpurun_out/sanitizer_$TOOL.log"
  [ "${PIPESTATUS[0]}" -ne 0 ] && rc=1
done
exit $rc
