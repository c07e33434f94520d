"""Builds libb200st.so in-tree with nvcc for sm_90a (no torch headers, plain C ABI).

Usage: python neurst_b200/csrc/build.py [--force]
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "libb200st.so")
OBJ = os.path.join(HERE, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _sources():
    return sorted(f for f in os.listdir(HERE) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(HERE)):
        if f.endswith((".cu", ".cuh", ".h")):
            h.update(f.encode())
            h.update(open(os.path.join(HERE, f), "rb").read())
    h.update(open(os.path.join(HERE, "..", "..", "include", "b200st.h"), "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def is_current():
    """True when the in-tree libb200st.so was built from exactly the sources (and flags) now in the tree."""
    stamp = os.path.join(OBJ, "digest.txt")
    return os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == _digest()


def build(force=False, verbose=False):
    """Builds under an exclusive file lock (all ranks of a torchrun job call this at import: one compiles, the others
    wait and find the library current) into temporary files that are os.replace()d into place, so no process can
    dlopen a half-written library.  A stale library next to a failed build raises (never loads silently)."""
    import fcntl
    os.makedirs(OBJ, exist_ok=True)
    if not force and is_current():
        return OUT
    with open(os.path.join(OBJ, ".lock"), "w") as lockf:
        fcntl.flock(lockf, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lockf, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    stamp = os.path.join(OBJ, "digest.txt")
    dig = _digest()
    if not force and is_current():       # another process built it while we waited for the lock
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError("libb200st.so is %s and nvcc (%s) is not available to rebuild it" %
                           ("stale (source digest mismatch)" if os.path.exists(OUT) else "missing", NVCC))
    srcs = _sources()

    def compile_one(src):
        obj = os.path.join(OBJ, src[:-3] + ".o")
        # per-source incremental build: recompile only when this source (or any header / the flags) changed
        h = hashlib.sha256(open(os.path.join(HERE, src), "rb").read())
        for f in sorted(os.listdir(HERE)):
            if f.endswith((".cuh", ".h")):
                h.update(open(os.path.join(HERE, f), "rb").read())
        h.update(open(os.path.join(HERE, "..", "..", "include", "b200st.h"), "rb").read())
        h.update(" ".join(FLAGS).encode())
        ostamp = obj + ".digest"
        if not force and os.path.exists(obj) and os.path.exists(ostamp) and open(ostamp).read() == h.hexdigest():
            return obj
        tmp = obj + ".tmp.%d" % os.getpid()
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(HERE, src), "-o", tmp]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        os.replace(tmp, obj)
        open(ostamp, "w").write(h.hexdigest())
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_one, srcs))
    tmp_out = OUT + ".tmp.%d" % os.getpid()
    cmd = [NVCC, "-shared", "-o", tmp_out] + objs + ["-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    os.replace(tmp_out, OUT)
    open(stamp, "w").write(dig)
    return OUT


IO_OUT = os.path.join(os.path.dirname(HERE), "libb200st_io.so")
IO_FLAGS = ["-O3", "-std=c11", "-fPIC", "-shared", "-Wall"]


def _io_digest():
    h = hashlib.sha256(open(os.path.join(HERE, "io_host.c"), "rb").read())
    h.update(open(os.path.join(HERE, "..", "..", "include", "b200st_io.h"), "rb").read())
    h.update(" ".join(IO_FLAGS).encode())
    return h.hexdigest()


def build_io(force=False):
    """libb200st_io.so: the host-side input-edge helpers (TFRecord framing, CRC-32C) — plain C, gcc, no CUDA."""
    import fcntl
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "io_digest.txt")
    dig = _io_digest()
    if not force and os.path.exists(IO_OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return IO_OUT
    with open(os.path.join(OBJ, ".lock_io"), "w") as lockf:
        fcntl.flock(lockf, fcntl.LOCK_EX)
        try:
            if not force and os.path.exists(IO_OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
                return IO_OUT
            tmp = IO_OUT + ".tmp.%d" % os.getpid()
            r = subprocess.run([os.environ.get("CC", "gcc")] + IO_FLAGS + [os.path.join(HERE, "io_host.c"), "-o", tmp],
                               capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("gcc failed for io_host.c:\n%s\n%s" % (r.stdout, r.stderr))
            os.replace(tmp, IO_OUT)
            open(stamp, "w").write(dig)
            return IO_OUT
        finally:
            fcntl.flock(lockf, fcntl.LOCK_UN)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_io(force="--force" in sys.argv))
