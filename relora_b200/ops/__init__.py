"""Hot-path operators.

``reference``  plain PyTorch (fp32-accumulating) definitions of every fused op — the numerics
               oracle for the CUDA kernels and the implementation used on CPU / gloo runs.
``native``     loader for the in-tree sm_90a extension (``relora_b200/_C*.so``).
``fused``      autograd functions over the native kernels.
``dispatch``   run-time switch between the two (CUDA + bf16 + extension present => native).
``quant``      block-scaled fp8 / fp4 storage of the frozen weights.
"""
