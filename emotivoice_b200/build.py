"""Builds libemotivoice_b200.so in-tree with nvcc for sm_90a (H100; no torch involved).

    python -m emotivoice_b200.build [--force]

The shared library is the product's only compute path; there is no CPU or eager
fallback.  It is git-ignored: build() makes it from the sources in every checkout.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libemotivoice_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "-cudart", "static"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    files = sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh"))
    files.append(os.path.join(INCLUDE, "emotivoice_b200.h"))
    for f in files:
        h.update(os.path.basename(f).encode())      # names, not absolute paths: a built tree may be moved
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def build(force=False, verbose=True):
    """Idempotent and safe to call from several processes at once (torchrun ranks): the check-and-compile
    section runs under an exclusive file lock, so one process compiles and the others then find the stamp.
    A current library is found without writing anything, so a built tree may be read-only."""
    import fcntl
    if not force and _up_to_date(_digest()):
        if verbose:
            print("emotivoice_b200.build: up to date, not recompiled", flush=True)
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _up_to_date(dig):
    stamp = os.path.join(LIB_DIR, "build.stamp")
    if not (os.path.exists(LIB_PATH) and os.path.exists(stamp)):
        return False
    with open(stamp) as f:
        return f.read().strip() == dig


def _build_locked(force, verbose):
    stamp = os.path.join(LIB_DIR, "build.stamp")
    dig = _digest()
    if not force and _up_to_date(dig):
        if verbose:
            print("emotivoice_b200.build: up to date (sources digest %s), not recompiled" % dig[:12], flush=True)
        return LIB_PATH
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIB_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc_path()] + NVCC_FLAGS + ["-I", INCLUDE, "-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    serialised = []
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed on %s" % src)
        if verbose and out.strip():
            print(out.decode())
        if b"C7520" in out:
            if not verbose:
                sys.stderr.write(out.decode())
            serialised.append(os.path.basename(src))
    if serialised:
        # such a binary computes the same results, but every MMA waits for the previous one to finish: refuse to build it
        raise RuntimeError("ptxas serialised wgmma instructions (warning C7520, reason above) in %s; a wgmma on a path ptxas cannot "
                           "prove warp-uniform is one cause" % ", ".join(serialised))
    cmd = [nvcc_path(), "-shared", "-o", LIB_PATH] + objs + ["-cudart", "static",
                                                           "-gencode", "arch=compute_90a,code=sm_90a"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(dig)
    if verbose:
        print("emotivoice_b200.build: compiled %d sources with nvcc for sm_90a (digest %s)" % (len(objs), dig[:12]), flush=True)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
