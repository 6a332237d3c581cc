"""Packaging for relora-b200.  The CUDA extension is built in-tree (``python -m relora_b200.csrc.build`` or
``python -c 'import __graft_entry__ as g; g.build()'``) rather than by setuptools, so that the same ``.so`` is used
from a checkout, from an editable install and on the GPU box the repository snapshot is shipped to."""
from setuptools import find_packages, setup

setup(
    name="relora_b200",
    version="0.1.0",
    description="Hopper-native (sm_90a) ReLoRA pre-training engine",
    packages=find_packages(include=["relora_b200", "relora_b200.*", "tools"]),
    package_data={"relora_b200": ["_C.so", "_data_helpers.so", "csrc/*.cu", "csrc/*.cuh", "csrc/*.h", "csrc/*.cpp"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.6", "numpy", "pyyaml"],
    extras_require={"full": ["transformers", "tokenizers", "datasets", "wandb", "loguru", "tqdm", "pybind11", "safetensors"]},
    license="Apache-2.0",
)
