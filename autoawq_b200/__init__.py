"""autoawq_b200: H100-native (sm_90a) AWQ W4A16 linear path behind the reference's module / extension API.

Layout: csrc/ (CUDA kernels + C ABI, built into lib/libb200awq.so), _cabi.py (ctypes binding),
ext.py (the `awq_ext` / `awq_v2_ext` operator surface), linear.py (WQLinear_* mirrors),
packing.py (packed-format producers), shard.py (column / row sharding across GPUs).
"""
__version__ = "0.1.0"
