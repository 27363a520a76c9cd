"""Install the unmodified reference package into oracle/_ref/ (git-ignored) for bench.py's reference arm.

The reference (daniabib/ComfyUI_ProPainter_Nodes) is pure Python with relative imports and has no installable
distribution metadata, so installing it is copying its package tree under the distribution's name:
oracle/_ref/comfyui_propainter_nodes/.  Nothing in it is edited, and the product never imports it.

The source is the directory named by PROPAINTER_REFERENCE, by default a checkout named `reference` next to this
repository.  Without a source, an existing install is kept (a tree that travels without the checkout still has it).
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PACKAGE = "comfyui_propainter_nodes"


def source_dir() -> str:
    return os.environ.get("PROPAINTER_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference"))


def install() -> str:
    """Copies the reference into oracle/_ref/<package>; returns what happened."""
    src, dst = source_dir(), os.path.join(REF_DIR, PACKAGE)
    if not os.path.isfile(os.path.join(src, "propainter_inference.py")):
        return "kept the existing install" if os.path.isdir(dst) else "no reference checkout found: not installed"
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    shutil.copytree(src, dst, ignore=shutil.ignore_patterns("examples", "*.pyc", "__pycache__", ".git*"))
    return "installed"


if __name__ == "__main__":
    print("reference:", install())
