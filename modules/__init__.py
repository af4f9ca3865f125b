"""Host-side mirror of the reference's ``modules`` package (taichi-dev/taichi-nerfs).

Same module / class / function names and call signatures as the reference, but every kernel is a
hand-written sm_90a CUDA kernel reached through the C-ABI library ``libngp_b200.so``
(include/ngp_b200.h) instead of a Taichi JIT kernel.
"""
