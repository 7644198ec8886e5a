#!/usr/bin/env bash
# compute-sanitizer passes over the small GPU paths (the mbarrier / wgmma / TMA-multicast code is where misuse would
# hide).  Run on an H100 with compute-sanitizer on PATH:
#     bash scripts/sanitize.sh > sanitize.log 2>&1
# Each tool first runs the smoke() encoder forward (wgmma GEMM + attention, LayerNorm, embed, pool); the later blocks run
# the small cases of the GPU tests that cover the GEMM epilogues (bias / residual / statistics / LayerNorm consumer /
# ordered split-K), both attention kernels, xsim (column filter, re-rank, list merge), the decoder step and beam search,
# and the speech kernels.  A clean run prints "ERROR SUMMARY: 0 errors" per tool.
set -u
cd "$(dirname "$0")/.."
for tool in memcheck racecheck synccheck; do
  echo "=== compute-sanitizer --tool $tool : smoke() ==="
  timeout 900 compute-sanitizer --tool "$tool" --print-limit 20 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -12
done
echo "=== compute-sanitizer --tool memcheck : pytest small decoder / speech / xsim cases ==="
timeout 1500 compute-sanitizer --tool memcheck --print-limit 20 python -m pytest -x -q -m gpu \
  tests/test_gpu_decoder.py::test_teacher_forced_steps_match_oracle \
  tests/test_gpu_speech.py::test_fbank_kernel_matches_oracle_and_golden \
  tests/test_gpu_speech.py::test_speech_encoder_vs_oracle tests/test_gpu_xsim.py::test_xsim_matches_oracle 2>&1 | tail -15
echo "=== compute-sanitizer --tool racecheck : speech encoder (rel-pos attention smem ring) + decoder step ==="
timeout 1500 compute-sanitizer --tool racecheck --print-limit 20 python -m pytest -x -q -m gpu \
  tests/test_gpu_speech.py::test_speech_encoder_vs_oracle \
  tests/test_gpu_decoder.py::test_teacher_forced_steps_match_oracle 2>&1 | tail -15
echo "=== compute-sanitizer --tool memcheck : skinny GEMM, fused-LayerNorm GEMM, graph-replayed beam search ==="
timeout 1500 compute-sanitizer --tool memcheck --print-limit 20 python -m pytest -x -q -m gpu \
  tests/test_gpu_kernels.py -k "skinny" \
  "tests/test_gpu_encoder.py::test_fused_layernorm_is_bitwise_the_separate_kernel" \
  tests/test_gpu_decoder.py::test_cuda_graph_replay_equals_eager_generation 2>&1 | tail -15
echo "=== memcheck: GEMM epilogues (bias / residual / statistics / LN consumer / split-K), attention ==="
timeout 360 compute-sanitizer --tool memcheck --print-limit 20 python -m pytest -x -q -m gpu tests/test_gpu_kernels.py \
  -k "(splitk and (700 or 2500)) or (residual_stats and (300 or 77)) or (ln_consumer and 130) or attention or (test_gemm_residual_fp32 and 515)" 2>&1 | tail -8
echo "=== memcheck: xsim (one direction, bidirectional, overflow, narrow spread), speech rel-pos attention on wgmma, decoder ==="
timeout 420 compute-sanitizer --tool memcheck --print-limit 20 python -m pytest -x -q -m gpu tests/test_gpu_xsim.py \
  tests/test_gpu_speech.py::test_relpos_attention_tcgen05_agrees_with_mma_sync_and_is_batch_invariant \
  tests/test_gpu_decoder.py -k "not large_slice" 2>&1 | tail -8
echo "=== racecheck: attention (wgmma), rel-pos attention (wgmma), xsim bidirectional small cases ==="
timeout 420 compute-sanitizer --tool racecheck --print-limit 20 python -m pytest -x -q -m gpu \
  tests/test_gpu_kernels.py tests/test_gpu_xsim.py \
  tests/test_gpu_speech.py::test_relpos_attention_tcgen05_agrees_with_mma_sync_and_is_batch_invariant \
  -k "attention_vs_sdpa or (bidir_matches and (64 or 5-3)) or relpos_attention" 2>&1 | tail -8
echo "=== synccheck: the same ==="
timeout 300 compute-sanitizer --tool synccheck --print-limit 20 python -m pytest -x -q -m gpu \
  tests/test_gpu_kernels.py tests/test_gpu_xsim.py \
  -k "attention_vs_sdpa or (bidir_matches and (64 or 5-3))" 2>&1 | tail -8
