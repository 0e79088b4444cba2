"""Recipe for the git-ignored oracle/_ref/: the original SC-SfMLearner project's Python modules, installed by
__graft_entry__.build() where a checkout of that project is available.  The original project is pure Python (no native
code to compile), so installing it is a copy of the modules that tests and bench.py's reference arms import: its
dataset classes and transforms (real-dataset loader tests), its train.py / models / losses (the stock PyTorch arms).

Source: $SCSFM_REFERENCE_DIR, else a checkout named `reference` next to this repository, else /root/reference.
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTALLED = os.path.join(ROOT, "oracle", "_ref")
FILES = ("train.py", "inverse_warp.py", "loss_functions.py", "logger.py", "utils.py", "custom_transforms.py", "models", "datasets")


def source():
    """The original project's checkout, or None."""
    for d in (os.environ.get("SCSFM_REFERENCE_DIR", ""), os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference"):
        if d and os.path.isfile(os.path.join(d, "datasets", "sequence_folders.py")):
            return os.path.abspath(d)
    return None


def install():
    """Copy the original project's modules into oracle/_ref/; a no-op where no checkout is available."""
    src = source()
    if src is None:
        return None
    os.makedirs(INSTALLED, exist_ok=True)
    for name in FILES:
        s, d = os.path.join(src, name), os.path.join(INSTALLED, name)
        if os.path.isdir(s):
            shutil.copytree(s, d, dirs_exist_ok=True, ignore=shutil.ignore_patterns("__pycache__"))
        elif os.path.exists(s):
            shutil.copyfile(s, d)
    return INSTALLED


def installed():
    """Directory holding the original project's modules ($SCSFM_REFERENCE_DIR or oracle/_ref/), or None."""
    for d in (os.environ.get("SCSFM_REFERENCE_DIR", ""), INSTALLED):
        if d and os.path.isfile(os.path.join(d, "datasets", "sequence_folders.py")):
            return os.path.abspath(d)
    return None
