"""Install the upstream ReLoRA package for ``bench.py --impl reference``.

    python oracle/install_reference.py /path/to/upstream/relora

Copies the upstream ``peft_pretraining`` package into ``oracle/_ref/`` (kept out of git), where the reference arm of bench.py
imports it from.  Nothing in the copy is edited.
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(ROOT, "oracle", "_ref")


def main(ref_root: str) -> None:
    src = os.path.join(ref_root, "peft_pretraining")
    if not os.path.isdir(src):
        sys.exit(f"{ref_root} has no peft_pretraining package")
    dst = os.path.join(DEST, "peft_pretraining")
    shutil.rmtree(dst, ignore_errors=True)
    shutil.copytree(src, dst, ignore=shutil.ignore_patterns("__pycache__"))
    print(dst)


if __name__ == "__main__":
    main(sys.argv[1])
