"""Loader for libgccb200.so -- the only compute path of this package.

There is deliberately NO fallback: if the CUDA library is missing or no sm_90
(Hopper) device is present, every compute entry point raises.  (The CPU oracle under
oracle/ is test infrastructure and is never imported from here.)
"""
import ctypes
import os

from . import _capi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgccb200.so")
_lib = None


class GccbError(RuntimeError):
    pass


def get():
    """The bound library handle; builds nothing, falls back to nothing."""
    global _lib
    if _lib is None:
        path = os.environ.get("GCCB200_LIB", LIB_PATH)     # developer knob: A/B a differently-tuned build
        if path != LIB_PATH:
            _lib = _capi.bind(ctypes.CDLL(path))
            return _lib
        if not os.path.exists(LIB_PATH):
            raise GccbError(
                "libgccb200.so not found at %s -- build it with `python -m gcc_b200.csrc.build` "
                "(or __graft_entry__.build()).  There is no CPU fallback." % LIB_PATH)
        _lib = _capi.bind(ctypes.CDLL(LIB_PATH))
    return _lib


def check(rc, what=""):
    if rc != _capi.GCCB_OK:
        msg = get().gccb_last_error()
        raise GccbError("%s failed (status %d): %s" % (what or "libgccb200 call", rc,
                                                      msg.decode() if msg else "?"))


_arch = None


def require_device():
    """Fail loudly unless a Hopper (compute capability 9.0) CUDA device is current."""
    global _arch
    if _arch is not None:
        return _arch
    import torch
    if not torch.cuda.is_available():
        raise GccbError("gcc_b200 needs a CUDA device (sm_90a); none is visible and there is "
                        "no CPU fallback.")
    arch = get().gccb_arch()
    if arch != 90:                    # sm_90a code loads on compute capability 9.0 only
        raise GccbError("gcc_b200 kernels are built for sm_90a only; current device reports "
                        "compute capability %s" % arch)
    _arch = arch
    return arch


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dptr(t):
    """Device pointer of a CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise GccbError("expected a CUDA tensor (no CPU path exists)")
    if not t.is_contiguous():
        raise GccbError("expected a contiguous tensor")
    return ctypes.c_void_p(t.data_ptr())
