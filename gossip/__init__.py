"""Drop-in alias: ``import gossip`` resolves to the H100-native implementation
with the reference's export list (``gossip/__init__.py:8-21``)."""
from stochastic_gradient_push_b200.parallel.ad_psgd import BilatGossipDataParallel
from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
from stochastic_gradient_push_b200.topology.graph_manager import (
    DynamicBipartiteExponentialGraph, DynamicBipartiteLinearGraph,
    DynamicDirectedExponentialGraph, DynamicDirectedLinearGraph, GraphManager,
    NPeerDynamicDirectedExponentialGraph, RingGraph)
from stochastic_gradient_push_b200.mixing_manager import MixingManager, UniformMixing
from stochastic_gradient_push_b200.gossiper import PushSum, PushPull
