"""invesalius3_b200 — H100-native (sm_90a) volumetric compute core for InVesalius 3.

Drop-in replacement for the per-voxel hot path (threshold, MIP/MIDA, flood fill, watershed,
marching cubes) behind the reference's numpy-in/numpy-out signatures:

  invesalius3_b200.invesalius_rs      mirror of the `invesalius_rs` package API
  invesalius3_b200.slice_ops          Slice threshold bodies
  invesalius3_b200.watershed_process  do_watershed
  invesalius3_b200.surface_process    marching cubes (create_surface_piece / contour)
  invesalius3_b200.device             the same ops on device-resident torch tensors
  invesalius3_b200.dist               Z-sharded multi-GPU versions (torch.distributed / NCCL)

All compute is hand-written CUDA in libb2v.so (C ABI: include/b2v.h). There is no CPU
fallback: importing a compute module without the built library or a CUDA device fails.
"""
__version__ = "0.1.0"
