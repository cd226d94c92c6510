"""Exception mapping for the C ABI error codes (mirrors the behaviour of
sourmash/src/sourmash/exceptions.py:58-75: codes 100 < c < 10000 raise ValueError)."""
from ._lowlevel import lib


class SourmashError(Exception):
    """Base error raised for failures reported by libsourmash_b200."""
    code = None

    def __init__(self, msg):
        Exception.__init__(self)
        self.message = msg
        self.rust_info = None

    def __str__(self):
        return self.message


class Panic(SourmashError):
    code = lib.SOURMASH_ERROR_CODE_PANIC


class CudaUnavailable(SourmashError):
    """The GPU path could not run (no device / CUDA failure).  There is no CPU fallback."""
    code = lib.SOURMASH_ERROR_CODE_CUDA


class IndexNotSupported(SourmashError):
    pass


def _exception_for(code):
    if code == lib.SOURMASH_ERROR_CODE_PANIC:
        return Panic
    if code == lib.SOURMASH_ERROR_CODE_CUDA:
        return CudaUnavailable
    if 100 < code < 10000:
        return ValueError
    return SourmashError
