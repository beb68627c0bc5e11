#!/bin/bash
# OSGP_IB: ResNet-50 / ImageNet, 90 epochs (recipe of the reference's job_scripts/submit_OSGP_IB.sh),
# re-targeted at 8xH100 nodes: ONE RANK PER GPU (the reference ran one process per
# 8-GPU node), NVLink/NVSwitch gossip inside a node.
#
#SBATCH --job-name=OSGP_IB
#SBATCH --output=OSGP_IB.out
#SBATCH --error=OSGP_IB.err
#SBATCH --nodes=NB_NODES
#SBATCH --ntasks-per-node=8
#SBATCH --cpus-per-task=12
#SBATCH --gres=gpu:8
#SBATCH --time=30:00:00
#
# Replace NB_NODES with the number of nodes; add --dataset_dir /path/to/imagenet
# (without it the run uses synthetic data) and --checkpoint_dir.
# SIGUSR1 90 s before the time limit -> checkpoint + requeue (ClusterManager):
#SBATCH --signal=USR1@90

# Gossip unit: by default every GPU is a gossip rank (8 x NB_NODES ranks).  Add
#   --nprocs_per_node 8
# to make the NODE the gossip unit, as in the reference (one 8-GPU node = one rank, batch 256):
# parameters are broadcast and gradients averaged inside the node through the NVSwitch (NVLS
# kernels), and only the nodes' first ranks gossip over the network.
export MASTER_ADDR=$(scontrol show hostnames "$SLURM_JOB_NODELIST" | head -n 1)
export HOSTNAME=$MASTER_ADDR

srun python -u gossip_sgd.py \
    --batch_size 32 --lr 0.1 --num_dataloader_workers 10 \
    --num_epochs 90 --nesterov True --warmup True \
    --push_sum True --graph_type 0 --overlap True --all_reduce False \
    --schedule 30 0.1 60 0.1 80 0.1 \
    --master_port 40100 --tag 'OSGP_IB_' --print_freq 100 --verbose False \
    --seed 1 --network_interface_type 'infiniband' \
    --checkpoint_dir results_dir/
