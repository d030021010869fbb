#!/bin/bash
# Configurations 3-5 on N GPUs: DDP vs ACCO side by side, Llama-3-1B (grad-accum 8) both arms, Llama-3-1B ACCO-ft SFT.
N=${1:-8}
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
mkdir -p results
timeout 200 $TR --master-port 29531 bench.py --gpus $N --steps 30 --warmup 5 --method ddp 2>&1 | grep "^{" > results/bench${N}_ddp.json; echo "ddp rc=$?"; cut -c1-200 results/bench${N}_ddp.json
timeout 300 $TR --master-port 29532 bench.py --gpus $N --steps 6 --warmup 3 --model llama3-1b --n-acc 8 2>&1 | grep "^{" > results/bench${N}_1b_ours.json; echo "1b ours rc=$?"; cut -c1-200 results/bench${N}_1b_ours.json
timeout 420 $TR --master-port 29533 bench.py --gpus $N --steps 6 --warmup 3 --model llama3-1b --n-acc 8 --impl reference 2>&1 | grep "^{" > results/bench${N}_1b_reference.json; echo "1b ref rc=$?"; cut -c1-200 results/bench${N}_1b_reference.json
mkdir -p /tmp/sft1b && cd /tmp/sft1b && timeout 420 $TR --master-port 29534 $OLDPWD/main.py train=acco-ft data=alpaca model=llama3-1b train.nb_steps_tot=$((N*2*10)) train.eval_step=$((N*2*6)) train.max_eval_batches=4 data.synthetic_docs=2048 train.tensorboard=False > $OLDPWD/results/sft1b_${N}.log 2>&1; echo "1b sft rc=$?"; cd $OLDPWD; grep -E "done:|eval loss|Error|error" results/sft1b_${N}.log | tail -5 | cut -c1-400; nvidia-smi --query-gpu=memory.used --format=csv,noheader | head -2
