#!/bin/bash
# One 8xH100 box, no scheduler: torchrun, one rank per GPU.
#   ./job_scripts/run_local_8gpu.sh sgp|osgp|dpsgd|ar|adpsgd [extra flags...]
set -euo pipefail
ALGO=${1:-sgp}; shift || true
NGPU=${NGPU:-8}
COMMON="--batch_size 32 --lr 0.1 --num_epochs 90 --nesterov True --warmup True \
  --schedule 30 0.1 60 0.1 80 0.1 --print_freq 100 --verbose False --seed 1 \
  --checkpoint_dir results_dir/ --tag ${ALGO}_"
case "$ALGO" in
  sgp)    SCRIPT=gossip_sgd.py;        FLAGS="--push_sum True --graph_type 0" ;;
  osgp)   SCRIPT=gossip_sgd.py;        FLAGS="--push_sum True --graph_type 0 --overlap True" ;;
  dpsgd)  SCRIPT=gossip_sgd.py;        FLAGS="--push_sum False --graph_type 1" ;;
  ar)     SCRIPT=gossip_sgd.py;        FLAGS="--all_reduce True --graph_type -1" ;;
  adpsgd) SCRIPT=gossip_sgd_adpsgd.py; FLAGS="--push_sum False --graph_type 1 --bilat True --train_fast True" ;;
  *) echo "unknown algorithm $ALGO"; exit 2 ;;
esac
exec python -m torch.distributed.run --nnodes=1 --nproc-per-node "$NGPU" \
  --master-addr 127.0.0.1 --master-port "${MASTER_PORT:-40100}" \
  "$SCRIPT" $COMMON $FLAGS "$@"
