#!/bin/bash
# compute-sanitizer over the kernel-level GPU tests (SURVEY.md §5 "race detection / sanitizers": the reference has none).
# Run on a GPU machine:   bash tools/sanitize.sh      (outputs under $SANITIZE_OUT, default sanitize_out/)
# memcheck: out-of-bounds / misaligned accesses; racecheck: shared-memory hazards between warps of a CTA; synccheck: invalid
# barrier usage.  The sanitizer serialises kernels and runs them 10-100x slower, so this takes the small-shape tests only
# (-k filters); wgmma / TMA kernels are exercised through test_gemm_plain / test_attn_prefill_tc / test_gemv_plain.
# NOT YET RUN: written after round 2's GPU budget was spent.
cd "$(dirname "$0")/.."
OUT="${SANITIZE_OUT:-sanitize_out}"
mkdir -p "$OUT"
SAN=/usr/local/cuda/bin/compute-sanitizer
SEL='test_norms or test_gemv_plain or test_gemv_fused or test_attn_decode or test_beam_topk or test_beam_step or test_sample_tokens or test_preprocess_image or test_image_to_uint8 or test_gemm_skinny'
TC='test_gemm_plain or test_attn_prefill_tc or test_conv3x3'
for tool in memcheck racecheck synccheck; do
  timeout 600 $SAN --tool $tool --error-exitcode 9 --print-limit 20 \
      python -m pytest tests/test_ops_gpu.py -x -q -k "$SEL" > "$OUT"/sanitize_${tool}.txt 2>&1
  echo "$tool (simt kernels) rc=$?"; tail -3 "$OUT"/sanitize_${tool}.txt
done
timeout 900 $SAN --tool memcheck --error-exitcode 9 --print-limit 20 \
    python -m pytest tests/test_ops_gpu.py -x -q -k "$TC" > "$OUT"/sanitize_memcheck_tc.txt 2>&1
echo "memcheck (wgmma / TMA kernels) rc=$?"; tail -3 "$OUT"/sanitize_memcheck_tc.txt
