"""In-tree build of the C-ABI CUDA library (sm_90a only).  (The oracle is pure Python / PyTorch: nothing to compile.)

    python -m allrank_b200.build            # or __graft_entry__.build()

nvcc cross-compiles without a GPU.  The resulting liballrank_b200.so stays in-tree (git-ignored), so the package is
importable from the repository tree.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "liballrank_b200.so")
STAMP = os.path.join(HERE, ".build_stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _fingerprint():
    h = hashlib.sha256()
    inc = os.path.join(os.path.dirname(HERE), "include", "allrank_b200.h")
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [inc, os.path.abspath(__file__)]
    for f in files:
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode())      # (not the absolute path: the tree moves between boxes)
            h.update(fh.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read() == fp:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in _sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {os.path.basename(src)}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
    link = [nvcc, "-shared", "-o", LIB] + objs
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    with open(STAMP, "w") as fh:
        fh.write(fp)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
