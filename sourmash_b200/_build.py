"""Build recipe for libsourmash_b200.so (nvcc, sm_90a only: H100).  Used by __graft_entry__.build().

Staleness is decided by CONTENT: a sha256 over every source, every header and the compiler flags is
stored next to the library (`libsourmash_b200.so.stamp`, git-ignored like the library).  File times do not
survive a copy of the tree to another machine, a hash does -- a prebuilt library that matches its sources is
used as it is instead of being recompiled in front of the first test."""
import glob
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsourmash_b200.so")
STAMP = LIB + ".stamp"
SOURCES = ["capi.cu", "sketch_kernels.cu", "compare_kernels.cu", "ingest.cu"]
PUBLIC_HEADER = os.path.join(HERE, "..", "include", "sourmash_b200.h")
OBJ_DIR = os.path.join(CSRC, "build")                 # git-ignored; only the linked .so ships
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC"]
LINK_LIBS = ["-lz", "-ldl"]


def headers():
    "every header a source may include: csrc/*.cuh, csrc/*.h and the public C header"
    found = sorted(glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")))
    return found + [PUBLIC_HEADER]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest(paths, extra=()):
    h = hashlib.sha256()
    for item in extra:
        h.update(item.encode() + b"\0")
    for p in paths:
        h.update(os.path.basename(p).encode() + b"\0")
        with open(p, "rb") as fh:
            h.update(fh.read())
        h.update(b"\0")
    return h.hexdigest()


def source_hash():
    "content hash of everything the library is compiled from"
    return _digest([os.path.join(CSRC, s) for s in SOURCES] + headers(), NVCC_FLAGS + LINK_LIBS)


def _object_hash(src):
    return _digest([os.path.join(CSRC, src)] + headers(), NVCC_FLAGS)


def _read(path):
    try:
        with open(path) as fh:
            return fh.read().strip()
    except OSError:
        return None


def built_hash():
    "the hash recorded when the present library was linked (None: no library / no stamp)"
    return _read(STAMP) if os.path.exists(LIB) else None


def needs_build():
    return built_hash() != source_hash()


def build(force=False, verbose=False):
    """One nvcc -c per source, side by side, then one link: a change to one file recompiles that file.
    Nothing is compiled when the stamp equals the hash of the sources, unless `force` or GRAFT_FORCE_BUILD."""
    force = force or bool(os.environ.get("GRAFT_FORCE_BUILD"))
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ_DIR, exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
        want = _object_hash(src)
        if not force and os.path.exists(obj) and _read(obj + ".stamp") == want:
            continue
        cmd = [nvcc_path()] + NVCC_FLAGS + ["-c", "-o", obj, src]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((cmd, obj, want, subprocess.Popen(cmd, cwd=CSRC)))
    for cmd, obj, want, p in procs:
        if p.wait() != 0:
            raise subprocess.CalledProcessError(p.returncode, cmd)
        with open(obj + ".stamp", "w") as fh:
            fh.write(want + "\n")
    cmd = [nvcc_path()] + NVCC_FLAGS + ["-shared", "-o", LIB] + \
        [os.path.join(OBJ_DIR, s[:-3] + ".o") for s in SOURCES] + LINK_LIBS
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd, cwd=CSRC)
    with open(STAMP, "w") as fh:
        fh.write(source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    build(force=True, verbose=True)
