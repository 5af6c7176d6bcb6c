set -x
OUT=${OUT:-results}; mkdir -p "$OUT"; export OUT      # output directory (git ignores results/)
nvidia-smi -L
python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 bench.py --gpus 2 --steps 120 --warmup 5 --no-cpu-baseline > $OUT/bench_train_n2.json 2> $OUT/bench_train_n2.err
tail -c 600 $OUT/bench_train_n2.json; tail -5 $OUT/bench_train_n2.err
python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29512 bench.py --gpus 2 --impl reference --steps 5 --warmup 1 2>&1 | tail -2 | cut -c1-300
