"""jellyfish_b200 -- H100-native (sm_90a) k-mer counting engine, drop-in for the `jellyfish count` path.

Package contents (only what the path needs):
  csrc/           sm_90a CUDA kernels + the C ABI (include/jfgpu.h) + the C++ host driver
  lib/            build products (libjfgpu.so, jellyfish-b200), made by __graft_entry__.build()
  _lib.py         ctypes declaration of the C ABI
  engine.py       Python mirror of the reference's hash_counter / dumper interfaces
  distributed.py  one-process-per-GPU sharded counting over torch.distributed
"""
from .engine import HashCounter, BloomCounter, ReadMerFile, JellyfishError, reference_matrix, mer_to_int, int_to_mer, canonical_int, load_database  # noqa: F401

__all__ = ["HashCounter", "BloomCounter", "ReadMerFile", "JellyfishError", "reference_matrix", "mer_to_int", "int_to_mer", "canonical_int", "load_database"]
