#!/bin/bash
# Multi-GPU verification on one box: parity tests (2 ranks: host collective, built-in NCCL, peer stores, one process / two
# devices), then bench.py under torchrun for every N given.  Usage: tools/multi_gpu_check.sh "2 4 8" [steps]
# SKIP_TESTS=1 / SKIP_P2P=1 leave out the parity tests / the peer-store bench line.  Writes multi_gpu_out/multi_*.{log,json}.
NS=${1:-2}
STEPS=${2:-300}
mkdir -p multi_gpu_out
if [ -z "$SKIP_TESTS" ]; then
  timeout 900 python -m pytest tests/test_gpu_multi.py -x -q -p no:cacheprovider 2>&1 | tail -15 > multi_gpu_out/multi_tests.log
  tail -5 multi_gpu_out/multi_tests.log
fi
port=29600
for n in $NS; do
  for sc in strong weak; do
    port=$((port + 1))
    timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $n --master-addr 127.0.0.1 --master-port $port \
      bench.py --gpus $n --steps $STEPS --warmup 10 --scaling $sc --no-secondary \
      > multi_gpu_out/multi_bench_n${n}_${sc}.json 2> multi_gpu_out/multi_bench_n${n}_${sc}.err
    echo "N=$n $sc rc=$?"; head -c 400 multi_gpu_out/multi_bench_n${n}_${sc}.json; echo; tail -2 multi_gpu_out/multi_bench_n${n}_${sc}.err
  done
  if [ -n "$SKIP_P2P" ]; then continue; fi
  port=$((port + 1))
  B200VIS_EXCHANGE=p2p timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $n --master-addr 127.0.0.1 --master-port $port \
    bench.py --gpus $n --steps $STEPS --warmup 10 --scaling strong --no-secondary \
    > multi_gpu_out/multi_bench_n${n}_strong_p2p.json 2> multi_gpu_out/multi_bench_n${n}_strong_p2p.err
  echo "N=$n strong p2p rc=$?"; head -c 300 multi_gpu_out/multi_bench_n${n}_strong_p2p.json; echo
done
