#!/bin/bash
# compute-sanitizer over a few tiny GPU tests (one attention, one GEMM, one state-machine case).
#   tools/run_sanitizer.sh <tool: memcheck|racecheck|synccheck|initcheck> <log> [pytest node ids...]
# Round-1 lesson: the first `import torch` on a fresh box takes ~1 min, longer than the sanitizer's default launch
# time-out ("No attachable process found") -> page the image in first and raise --launch-timeout.
# Round-2 lesson: the pass over the kernels BEFORE programmatic dependent launch was extended is clean; a second pass over the final kernels -- every glue kernel launched with the programmatic
# attribute, griddepcontrol in the attention kernel, st.shared::cluster merge, Philox sampling kernel -- took the GPU box
# down twice (box lost ~3 min into memcheck, nothing returned).  The runner therefore switches PDL off; do not point it
# at PDL launches on a shared box.
export LADE_PDL=0 LADE_PDL_GLUE=0
set -u
TOOL=${1:-memcheck}; LOG=${2:-gpurun_out/sanitizer_$TOOL.log}; shift 2 || true
if [ $# -eq 0 ]; then
  set -- "tests/test_gpu_attention.py::test_attention_steady_shapes_vs_oracle[64-15-5-15-2-2-5-2]" \
         "tests/test_gpu_attention.py::test_attention_prefill_causal_vs_oracle[300-2-2-3-2]" \
         "tests/test_gpu_state_machine.py::test_device_state_machine_matches_reference_trace[tiny_bf16_w5n3g3]" \
         "tests/test_gpu_gemm.py::test_gemm_matches_fp32_reference[120-1000-1024-64-2]" \
         "tests/test_gpu_layer_ops.py"
fi
python -c "import torch; torch.zeros(1).cuda()" >/dev/null 2>&1
SAN=$(command -v compute-sanitizer || echo /usr/local/cuda/bin/compute-sanitizer)
timeout ${SAN_TIMEOUT:-900} "$SAN" --tool "$TOOL" --target-processes all --launch-timeout 600 \
    --error-exitcode 97 --print-limit 40 ${SAN_EXTRA:-} \
    python -m pytest -x -q -m gpu -p no:cacheprovider "$@" > "$LOG" 2>&1
rc=$?
echo "sanitizer $TOOL rc=$rc" >> "$LOG"
grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|rc=" "$LOG" | tail -5
exit 0
