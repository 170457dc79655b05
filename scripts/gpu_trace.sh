# On the GPU machine: per-team wait/busy breakdown of the fused kernel (diagnosis build -DLEXP_TRACE=1 from scripts/build_variants.py).
#   bash scripts/gpu_trace.sh [trace]
cd "$(dirname "$0")/.." || exit 1
V=${1:-trace}
mkdir -p gpurun_out
ORIG=$(mktemp)
cp localexpstereo_b200/liblexp_cuda.so "$ORIG"
trap 'cp "$ORIG" localexpstereo_b200/liblexp_cuda.so; rm -f "$ORIG"' EXIT   # the shipped library comes back however the run ends
cp variants/liblexp_cuda_$V.so localexpstereo_b200/liblexp_cuda.so
rm -f gpurun_out/trace.txt
LEXP_TRACE_FILE=gpurun_out/trace.txt timeout 600 python bench.py --steps 1 --warmup 3 --no-graph --no-cpu-baseline > gpurun_out/trace_bench.log 2>&1
python scripts/trace_summary.py gpurun_out/trace.txt | tee gpurun_out/trace_summary_$V.txt
