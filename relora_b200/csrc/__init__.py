"""sm_90a sources of the in-tree extension ``relora_b200/_C.so`` (+ the host C++ data helpers).

    gemm_wgmma.cu     persistent TMA + wgmma GEMM (LoRA K-extension, split-K, fp8), LoRA input-gradient kernel
    attention.cu      causal flash attention forward / dQ / dK,dV on wgmma
    norm_warp.cu      RMSNorm forward (+ dropout-expanded copies) / backward
    elementwise.cu    dropout expand / combine, SwiGLU, embedding, transpose, hash re-init
    rope.cu           rotary embedding (Llama layout), fused dq/dk/dv pack + inverse rotation
    neox.cu           GPT-NeoX / Pythia block: LayerNorm, GELU, partial rotary on the fused qkv layout
    loss.cu           in-place softmax cross-entropy forward + backward
    optim.cu          fused AdamW on flat buffers, Σx², moment pruning (random / exact magnitude quantile)
    fp8.cu            per-tensor E4M3 / E5M2 quantisation for the kind::f8f6f4 path
    comm.cu           NVLink peer-memory collectives (P2P + multimem): all-reduce, fused reduce-scatter / clip / AdamW / all-gather
    bindings.cpp      pybind11 / torch::Tensor glue;  data_helpers.cpp  index-map builders of the NeoX data pipeline

Build: ``python -m relora_b200.csrc.build`` (nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo; cross-compiles without a GPU).
"""
from .build import CPP_SOURCES, CUDA_SOURCES, HEADERS, build  # noqa: F401
