#!/bin/bash
# N-GPU machine (bash scripts/multi_gpu_check.sh [N] [output dir]): bench under torchrun, the recursive-evaluation CLI under
# torchrun, data generation with one locker per GPU.
N=${1:-2}
O=${2:-multi_gpu_check_out}; mkdir -p $O
timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29531 bench.py --gpus $N --steps 3 --warmup 3 --no-cpu-baseline > $O/bench_n$N.json 2> $O/bench_n$N.err
python - <<PY
import json
d = json.loads(open("$O/bench_n$N.json").read().strip().splitlines()[-1])
print("bench N=$N", d["value"], d["ms_per_step"], d["e2e"]["value"], d["n_gpus"], d["clocks"]["sm_mhz"])
PY
tail -2 $O/bench_n$N.err
timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29532 -m rebel_b200.recursive_eval --num_dice 2 --num_faces 3 --subgame_iters 1024 --cfr --no_full_tree --num_repeats 256 --batch_repeats 128 --random_net_seed 0 2>&1 | tail -1 | cut -c1-500
timeout 100 python -m rebel_b200.recursive_eval --num_dice 1 --num_faces 4 --subgame_iters 1024 --cfr --num_repeats 0 2>&1 | tail -4
timeout 200 python scripts/datagen_bench.py --devices $N --threads 2 --games 8192 --seconds 12 --warmup 4 2>&1 | tail -1
