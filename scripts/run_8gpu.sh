#!/bin/bash
# Single 8xH100 box without Slurm.
#   scripts/run_8gpu.sh                                   # train=acco data=openwebtext model=llama125m
#   NGPU=4 scripts/run_8gpu.sh train=dpu model=llama3-1b
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/.." && pwd)"     # artefacts (checkpoints/, tensorboard/, results.csv) land in the CALLER's directory
if [ "$#" -eq 0 ]; then
    set -- train=acco data=openwebtext model=llama125m
fi
exec python -m torch.distributed.run --nnodes=1 --nproc-per-node "${NGPU:-8}" --master-addr 127.0.0.1 --master-port "${PORT:-29500}" \
    "$ROOT/main.py" "$@"
