#!/bin/bash
# N GPUs of one box: exchange paths bit for bit, then the bench with the p2p exchange and with the NCCL all-gather.
#   bash tools/gpu_multi.sh 2
N=${1:-2}
mkdir -p gpurun_out
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
timeout 600 $TR --master-port 29511 tools/check_exchange.py > gpurun_out/n${N}_exchange.log 2>&1
timeout 900 $TR --master-port 29512 bench.py --gpus $N --steps 32 --warmup 3 --no-cpu-baseline > gpurun_out/n${N}_bench.json 2> gpurun_out/n${N}_bench.err
timeout 900 $TR --master-port 29513 bench.py --gpus $N --steps 32 --warmup 3 --no-cpu-baseline --no-extra-configs --exchange allgather > gpurun_out/n${N}_bench_allgather.json 2> gpurun_out/n${N}_bench_allgather.err
tail -6 gpurun_out/n${N}_exchange.log; tail -c 800 gpurun_out/n${N}_bench.err; grep "^{" gpurun_out/n${N}_bench.json | head -c 300; echo; grep "^{" gpurun_out/n${N}_bench_allgather.json | head -c 300
