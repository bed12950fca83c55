#!/bin/bash
# the round's 2-GPU evidence: C++ sharded aggregator, the full bench line at N=2 (e2e per rank, exchange checked,
# config-5 ride-along path forced on), reference arm at N=2, sharded rank/select
mkdir -p gpurun_out
nvidia-smi topo -m > gpurun_out/topo_n2.txt 2>&1
timeout 600 python -m pytest tests -m gpu -q -k "sharded" 2>&1 | tail -3 | tee gpurun_out/pytest_n2.log
timeout 300 bash scripts/run_sharded_cxx.sh 2>&1 | grep "OK\|FAIL" | tee gpurun_out/sharded_cxx_nccl.log
P=30117
BENCH_C5_WORLD=2 timeout 1800 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $P bench.py --gpus 2 --steps 20 --warmup 5 2> gpurun_out/bench_c3_n2.err | tail -1 | tee gpurun_out/bench_c3_n2.json | cut -c1-300
tail -c 400 gpurun_out/bench_c3_n2.err
timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $((P+1)) bench.py --impl reference --gpus 2 --steps 3 --warmup 1 2>/dev/null | tail -1 | tee gpurun_out/bench_ref_n2.json | cut -c1-200
timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $((P+2)) bench.py --gpus 2 --workload c5 --no-e2e --steps 10 2> gpurun_out/bench_c5_n2.err | tail -1 | tee gpurun_out/bench_c5_n2.json | cut -c1-200
timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $((P+3)) scripts/bench_c4_sharded.py 2>&1 | tail -1 | tee gpurun_out/bench_c4_n2.json | cut -c1-200
