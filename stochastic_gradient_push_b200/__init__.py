"""
stochastic_gradient_push_b200 -- H100-native gossip-SGD (SGP / OSGP / D-PSGD /
AD-PSGD / AllReduce-SGD) with the API surface of
facebookresearch/stochastic_gradient_push (``gossip/__init__.py:8-21``).
"""

from .topology import (
    GraphManager, Edge,
    DynamicDirectedExponentialGraph, NPeerDynamicDirectedExponentialGraph,
    DynamicBipartiteExponentialGraph, DynamicDirectedLinearGraph,
    DynamicBipartiteLinearGraph, RingGraph, GRAPH_TOPOLOGIES)
from .mixing_manager import (MixingManager, UniformMixing, SelfWeightedMixing,
                             MIXING_STRATEGIES)
from .gossiper import Gossiper, PushSum, PushPull, BilatPushPull

__version__ = '0.1.0'


def __getattr__(name):
    # heavy wrappers are imported lazily so that the pure-math layers stay
    # importable without torch.distributed / CUDA
    if name == 'GossipDataParallel':
        from .parallel.distributed import GossipDataParallel
        return GossipDataParallel
    if name == 'BilatGossipDataParallel':
        from .parallel.ad_psgd import BilatGossipDataParallel
        return BilatGossipDataParallel
    if name == 'AllReduceDataParallel':
        from .parallel.allreduce import AllReduceDataParallel
        return AllReduceDataParallel
    raise AttributeError(name)
