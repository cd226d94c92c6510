"""cffi ABI-mode binding of libsourmash_b200.so -- the same mechanism the reference uses
for its Rust cdylib (maturin ``bindings = "cffi"`` generates ``sourmash/_lowlevel`` which
dlopen()s the library; sourmash/pyproject.toml:138-155, src/sourmash/utils.py:3).

Exports ``ffi`` and ``lib`` like the reference's ``sourmash._lowlevel``.  The library must
have been built (``python -m sourmash_b200._build`` / ``__graft_entry__.build()``); there is
deliberately no fallback if it is missing.
"""
import os
import re

import cffi

_HERE = os.path.dirname(os.path.abspath(__file__))
_HEADER = os.path.join(os.path.dirname(_HERE), "include", "sourmash_b200.h")
LIB_PATH = os.path.join(_HERE, "libsourmash_b200.so")


def _cdef_source():
    with open(_HEADER) as fh:
        text = fh.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    lines = []
    for line in text.splitlines():
        s = line.strip()
        if s.startswith("#") or s.startswith('extern "C"') or s == "}":
            continue
        lines.append(line)
    return "\n".join(lines)


ffi = cffi.FFI()
ffi.cdef(_cdef_source())

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build the CUDA library first "
        "(python -m sourmash_b200._build); sourmash_b200 has no pure-Python/CPU fallback")

lib = ffi.dlopen(LIB_PATH)
ffi.init_once(lib.sourmash_init, "init")


def declared_symbols():
    """Every function name declared in include/sourmash_b200.h."""
    src = _cdef_source()
    return sorted(set(re.findall(r"\b([a-z_][a-z0-9_]*)\s*\(", src)) - {"void"})
