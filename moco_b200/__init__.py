"""moco_b200 -- H100-native MoCo contrastive hot path behind bl0/moco's own API.

    from moco_b200.NCE import MemoryMoCo, NCESoftmaxLoss     # moco.NCE
    from moco_b200.util import DistributedShufle, dist_collect  # moco.util

Device work is done by hand-written sm_90a kernels in ``libmoco_b200.so``
(C ABI: ``include/moco_b200.h``); see INTEGRATION.md.
"""
__version__ = "0.1.0"
