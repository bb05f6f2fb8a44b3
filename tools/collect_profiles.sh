#!/bin/bash
# Runs on a GPU machine: ncu captures, launch list, sanitizer logs and variant benches, written to profile_out/.
# usage: bash tools/collect_profiles.sh
O=profile_out
mkdir -p $O
NCU="ncu --set full --clock-control none --import-source on"
# 1. dominant kernel, 2^20 Merkle4 digests: skip the 3 warm-up launches, capture the first timed one
timeout 600 $NCU -k regex:k_sponge_digest -s 3 -c 1 -f -o $O/r2_prof_merkle4 python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-tree > $O/ncu_merkle4.log 2>&1
# 2. raw permutation kernel and decrypt kernel
timeout 600 $NCU -k regex:k_permute -s 3 -c 1 -f -o $O/r2_prof_permute python bench.py --workload permute --steps 2 --warmup 3 --no-cpu-baseline > $O/ncu_permute.log 2>&1
timeout 600 $NCU -k regex:k_crypt -s 3 -c 1 -f -o $O/r2_prof_decrypt python bench.py --workload decrypt --steps 2 --warmup 3 --no-cpu-baseline > $O/ncu_decrypt.log 2>&1
# 3. opening verification kernel (depth 10, arity 4) and the lane-split small-batch kernel
timeout 600 $NCU -k regex:k_merkle_verify -c 1 -f -o $O/r2_prof_verify python tools/profile_aux.py verify > $O/ncu_verify.log 2>&1
timeout 600 $NCU -k regex:k_sponge_digest_coop -s 1 -c 1 -f -o $O/r2_prof_coop python tools/profile_aux.py coop > $O/ncu_coop.log 2>&1
# 4. launch list of the default bench command (times are cold-cache and serialised: shares only)
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file $O/r2_launches_bench_merkle4.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline > $O/ncu_launches.log 2>&1
# 5. sanitizers on the new kernels (small shapes)
timeout 900 compute-sanitizer --tool memcheck python -m pytest tests/test_gpu_merkle_open.py -m gpu -q -x -k "device or mirror" > $O/r2_sanitizer_memcheck.log 2>&1
timeout 900 compute-sanitizer --tool racecheck python -m pytest tests/test_gpu_merkle_open.py -m gpu -q -x -k "device" > $O/r2_sanitizer_racecheck.log 2>&1
# 6. north_star's shared-memory/TMA staging of the round tables vs the constant bank (receipt for the deviation)
python bench.py --steps 20 --warmup 5 --no-cpu-baseline --no-tree > $O/r2_bench_const_bank.json 2>/dev/null
P252_NVCC_EXTRA="-DP252_CONST_SMEM=1" python -m poseidon252_b200.build --force > /dev/null 2>&1 && \
  python bench.py --steps 20 --warmup 5 --no-cpu-baseline --no-tree > $O/r2_bench_const_smem.json 2>/dev/null
python -m poseidon252_b200.build --force > /dev/null 2>&1
ls -la $O | tail -30
