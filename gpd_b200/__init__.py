"""gpd_b200 — the grasp-candidate hot path of atenpas/gpd on H100 (sm_90a).

The product is the C-ABI library gpd_b200/libgpd_b200.so (include/gpd_b200.h); this package is its ctypes binding
(`lib`), the ctypes mirror of the boundary structs (`abi`), seeded input generators (`scenes`) and the multi-GPU
plumbing (`sharding`). Nothing here computes on the CPU: without the built library `lib` raises.
"""
__version__ = "0.1.0"
