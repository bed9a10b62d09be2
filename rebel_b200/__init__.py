"""rebel_b200 — H100-native CFR self-play data generation for ReBeL / Liar's Dice (hot path only).

Layers: CUDA kernels + C ABI (csrc/, libcfrb200.so, include/cfrb200.h) -> ctypes binding (capi.py) and the C++
`rela` pybind module mirroring the reference's cfvpy.rela surface -> models.py (PyTorch Net2, Python side only).
"""
from . import capi, models  # noqa: F401
from .capi import NET_FP32, NET_TC_CLUSTER, NET_TC_F16, NET_TC_F16X2, NET_ZERO, SOLVER_CFR, SOLVER_FP, STATE_F32, STATE_F64, CfrbError, WaveSolver, tc_cluster_net_supported  # noqa: F401
