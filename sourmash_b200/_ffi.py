"""Calling convention of the C ABI, Python side.

The library reports failures through a thread-local (code, message) slot instead of return
codes (include/sourmash_b200.h; same protocol as the reference's FFI, whose Python half is
sourmash/src/sourmash/utils.py:9-78).  ``rustcall`` wraps one call in
clear-slot / call / poll-slot / raise; ``RustObject`` owns an opaque handle and frees it with
the class's ``__dealloc_func__``.  The names are kept so code written against the reference's
helpers keeps working.
"""
from ._lowlevel import ffi, lib
from .exceptions import _exception_for


def decode_str(sstr, free=True):
    "SourmashStr (returned by value) -> str; owned buffers are released."
    try:
        if sstr.data == ffi.NULL or not sstr.len:
            return ""
        return bytes(ffi.buffer(sstr.data, sstr.len)).decode("utf-8", "replace")
    finally:
        if free and sstr.owned:
            lib.sourmash_str_free(ffi.new("SourmashStr *", sstr))


def _raise_pending_error():
    code = lib.sourmash_err_get_last_code()
    if code:
        message = decode_str(lib.sourmash_err_get_last_message())
        lib.sourmash_err_clear()
        raise _exception_for(code)(message)


def rustcall(func, *args):
    "Call into the library and convert a recorded error into the mapped Python exception."
    lib.sourmash_err_clear()
    result = func(*args)
    _raise_pending_error()
    return result


class RustObject:
    "Base class of the Python objects that wrap an opaque library handle."

    __dealloc_func__ = None
    _objptr = None
    _shared = False          # True: the handle belongs to someone else, never free it

    def __init__(self):
        raise TypeError(f"Cannot instantiate {type(self).__name__!r} objects")

    @classmethod
    def _from_objptr(cls, ptr, shared=False):
        obj = object.__new__(cls)
        obj._objptr, obj._shared = ptr, shared
        return obj

    def _get_objptr(self):
        if not self._objptr:
            raise RuntimeError("Object is closed")
        return self._objptr

    def _methodcall(self, func, *args):
        return rustcall(func, self._get_objptr(), *args)

    def __del__(self):
        ptr, self._objptr = self._objptr, None
        release = type(self).__dealloc_func__
        if ptr is not None and not self._shared and release is not None and lib is not None:
            release(ptr)
