"""b200cast: the GraphCast 6 h step and rollout on NVIDIA H100 (sm_90a).

The compute path is `libgraphcast_b200.so` (hand-written CUDA behind the C ABI of
`include/graphcast_b200.h`); the modules of this package mirror the reference's Python surface for
that path (`graphcast`, `rollout`, `normalization`, `casting`, `autoregressive`, `checkpoint`, …) and
add the multi-GPU drivers (`partitioned`, `parallel`).  There is no CPU fallback: importing the
package is cheap, constructing a model without the library or without CUDA raises.
"""

__version__ = "0.2.0"
