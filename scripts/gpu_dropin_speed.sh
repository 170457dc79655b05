# On the GPU machine: the reference's UNCHANGED OpenMP loop (oracle/dropin_check.cpp, compiled from the reference headers) with the
# CUDA adapter installed, at a realistic size and with all host threads: correctness of every call against the reference CPU
# energy, how many calls the library combined into batched launches, and the thread-seconds spent in each energy.
#   bash scripts/gpu_dropin_speed.sh
cd "$(dirname "$0")/.." || exit 1
mkdir -p gpurun_out
T=$(nproc)
for args in "--threads $T --W 1024 --H 768 --D 64 --K 3" "--batched --W 1024 --H 768 --D 64 --K 3" "--threads 1 --W 512 --H 384 --D 64 --K 2" "--naive --threads $T --W 450 --H 375 --D 64 --K 3"; do
  echo "== dropin_check $args"
  timeout 800 ./oracle/_ref/dropin_check $args
done 2>&1 | tee gpurun_out/dropin_speed.txt
