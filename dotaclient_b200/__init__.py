"""dotaclient_b200 -- CUDA-native (H100) implementation of DotaClient's distributed-optimizer hot path.

Drop-in module surface of the reference (TimZaman/dotaclient @ 8615b90):

* ``dotaclient_b200.policy``       <-> reference ``policy.py``       (``Policy``, ``REWARD_KEYS``, ``eps``)
* ``dotaclient_b200.optimizer``    <-> reference ``optimizer.py``    (``DotaOptimizer``, ``Sequence``, ``MessageQueue``,
  ``advantage_returns``, ``discount``, ``init_distribution``, ``main``)
* ``dotaclient_b200.distributed``  <-> reference ``distributed.py``  (``DistributedDataParallelSparseParamCPU``)

The arithmetic runs in hand-written sm_90a CUDA kernels behind the C-ABI declared in
``include/dotaclient_b200.h`` (``dotaclient_b200/csrc``).  There is no CPU fallback.
"""
__version__ = "0.1.0"
