"""Stage the UNMODIFIED reference under oracle/_ref/ (TEST / BASELINE INFRASTRUCTURE ONLY).

The reference (hahnyuan/PTQ4ViT) is pure Python with no setup.py / pyproject, so "installing" it is a copy of its
importable packages.  `__graft_entry__.build()` runs this recipe; oracle/_ref/ is git-ignored (never part of this
repository's history) and belongs to the built tree, so a machine that runs the GPU tests needs only the build output.
It is used by
  * oracle/ref_harness.py -- tests/test_reference_gpu.py, test_calibrator_gpu.py, test_conv_gpu.py, test_integer_gpu.py
    run the reference classes on the GPU next to the CUDA path; tests/test_reference_harness_cpu.py on the CPU;
  * bench.py               -- `--impl reference` (CPU arm) and the `reference_gpu` comparator.
Nothing under ptq4vit_b200/ imports it.

    python oracle/stage_ref.py            # copies from $PTQ4VIT_REFERENCE (default /root/reference)
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(ROOT, "oracle", "_ref")
PACKAGES = ("quant_layers", "utils", "configs")


def stage(src=None, quiet=False):
    """Copy the reference's importable packages; returns DEST, or None when no reference tree is available (an already
    staged copy is kept)."""
    src = src or os.environ.get("PTQ4VIT_REFERENCE", "/root/reference")
    if not all(os.access(os.path.join(src, pkg), os.R_OK | os.X_OK) for pkg in PACKAGES):
        return DEST if os.path.isdir(os.path.join(DEST, "quant_layers")) else None
    os.makedirs(DEST, exist_ok=True)
    for pkg in PACKAGES:
        dst = os.path.join(DEST, pkg)
        if os.path.isdir(dst):
            shutil.rmtree(dst)
        # plain copies (no mode bits): the staged tree stays writable for whoever rebuilds or cleans it
        shutil.copytree(os.path.join(src, pkg), dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"),
                        copy_function=shutil.copyfile)
    if not quiet:
        print(f"staged {', '.join(PACKAGES)} from {src} into {DEST}")
    return DEST


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
