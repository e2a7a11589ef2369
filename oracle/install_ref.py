"""Copies the reference's ``mbrl`` package (facebookresearch/mbrl-lib, pure Python) from a checkout into ``oracle/_ref``,
where the CPU bench arm, the golden-vector generator and the reference-object tests import it from.  ``oracle/_ref`` is
git-ignored: the reference is not part of this project.  ``build()`` runs this when a checkout is found (``MBRL_LIB_SRC``,
else ``DEFAULT_SRC``); without one the reference-object tests skip.

    python oracle/install_ref.py [PATH_TO_MBRL_LIB_CHECKOUT]
"""
import os
import shutil
import sys

DEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
DEFAULT_SRC = "/root/reference"  # where the build hosts keep the mbrl-lib checkout


def source() -> str:
    return os.environ.get("MBRL_LIB_SRC", DEFAULT_SRC)


def install(src: str) -> str:
    pkg = os.path.join(src, "mbrl")
    if not os.path.isdir(pkg):
        raise SystemExit(f"{src} has no mbrl/ package")
    shutil.rmtree(DEST, ignore_errors=True)
    shutil.copytree(pkg, os.path.join(DEST, "mbrl"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    return DEST


def install_if_available():
    """Returns oracle/_ref after copying the reference into it, or None when no readable checkout is found."""
    src = source()
    try:
        if not os.path.isdir(os.path.join(src, "mbrl")):
            return None
    except OSError:
        return None
    return install(src)


if __name__ == "__main__":
    print(install(sys.argv[1] if len(sys.argv) > 1 else source()))
