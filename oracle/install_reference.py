"""Install the UNMODIFIED reference package into oracle/_ref (git-ignored) -- TEST / BENCH INFRASTRUCTURE, run where
an allRank source tree is available ($ALLRANK_REFERENCE, default /root/reference).

    python oracle/install_reference.py

Recipe: pip install --no-index --no-build-isolation --no-deps --target oracle/_ref <copy of the source tree in a
temporary directory>  (the source tree may be read-only; its pinned dependency versions -- torch 1.13, numpy <= 1.21
... -- are not what this project runs on, hence --no-deps; the three missing pure-Python dependencies are the stubs in
oracle/_stubs).  Nothing of the reference enters the repository: oracle/_ref is listed in .gitignore.
"""
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.environ.get("ALLRANK_REFERENCE", "/root/reference")
TARGET = os.path.join(ROOT, "oracle", "_ref")


def installed():
    return os.path.isfile(os.path.join(TARGET, "allrank", "main.py"))


def install(force=False):
    if installed() and not force:
        return TARGET
    if not os.path.isdir(os.path.join(REF_SRC, "allrank")):
        raise RuntimeError(f"no allRank source tree at {REF_SRC} (set ALLRANK_REFERENCE)")
    shutil.rmtree(TARGET, ignore_errors=True)
    os.makedirs(TARGET, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="allrank_src_")
    try:
        src = os.path.join(tmp, "reference")
        shutil.copytree(REF_SRC, src, ignore=shutil.ignore_patterns(".git", "__pycache__"))
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
               "--target", TARGET, src]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0 or not installed():
            # last resort: the package is pure Python -- copy the package directory as it is
            shutil.copytree(os.path.join(REF_SRC, "allrank"), os.path.join(TARGET, "allrank"), dirs_exist_ok=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return TARGET


def import_path():
    """sys.path entries that make `import allrank` resolve to oracle/_ref behind the three stub modules."""
    return [os.path.join(ROOT, "oracle", "_stubs"), TARGET]


if __name__ == "__main__":
    print(install(force="--force" in sys.argv))
