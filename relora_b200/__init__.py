"""relora_b200 — a Hopper (sm_90a) native ReLoRA pre-training engine.

Layout
------
config      CLI / YAML surface (same flags as the reference ``torchrun_main.py``)
relora      ReLoRaLinear / ReLoRaModel, jagged schedulers, optimizer-state resets
models      Llama and Pythia (GPT-NeoX) with HF-compatible parameter names
ops         hot-path operators: PyTorch fp32 references + sm_90a CUDA kernels
parallel    flat parameter store, NCCL baseline and NVLink peer-memory collectives
engine      training loop, fused train step (CUDA graphs), evaluation
data        HF-disk, synthetic and NeoX/Megatron mmap datasets (C++ index builders)
ckpt        reference-layout checkpoints, autoresume
obs         logging / metrics / profiler glue
"""

__version__ = "0.1.0"
