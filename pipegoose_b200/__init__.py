"""pipegoose_b200 — a Hopper (H100, sm_90a) native 3D-parallel training library with the
capabilities and user-facing API of xrsrke/pipegoose.

Python orchestrates; the hot ops are hand-written sm_90a CUDA kernels in ``pipegoose_b200/csrc``
(wgmma GEMMs fed by TMA and fused with their NVLink collectives), loaded from the in-tree
extension ``pipegoose_b200/_C.so`` (see ``pipegoose_b200.ops``).
"""

__version__ = "0.2.0"
