"""ctypes binding of libb200wave.so (the C ABI declared in include/b200wave.h).

There is deliberately NO fallback: if the CUDA library has not been built, or a tensor is not a
CUDA float32 tensor, the call raises.  (The CPU oracle under oracle/ is test infrastructure and
is never imported from here.)
"""
import ctypes
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200W_LIB: load an experimental build of the same library instead (tools/ab.py times one); still CUDA-only.
SO_PATH = os.environ.get('B200W_LIB') or os.path.join(_HERE, 'libb200wave.so')
_lib = None

c_ll = ctypes.c_longlong
c_vp = ctypes.c_void_p
c_int = ctypes.c_int

# every symbol include/b200wave.h declares (tests/test_abi.py checks the library exports them all)
SYMBOLS = [
    'b200w_version', 'b200w_strerror', 'b200w_last_cuda_error', 'b200w_dwt_coeff_len', 'b200w_dwt_rec_len',
    'b200w_dwt_afb2d', 'b200w_dwt_sfb2d', 'b200w_dtcwt_fwd_j1', 'b200w_dtcwt_fwd_j2plus', 'b200w_dtcwt_inv_j1',
    'b200w_dtcwt_inv_j2plus', 'b200w_scat_j1', 'b200w_dwt_forward',
]
KERNEL_ENTRIES = SYMBOLS[5:13]
# float64: the generic tile kernels and the 1-D row kernels instantiated for double (csrc/b200wave.cu, csrc/dwt1d.cu)
F64_ENTRIES = ['b200w_dwt_afb2d', 'b200w_dwt_sfb2d', 'b200w_dwt_afb1d', 'b200w_dwt_sfb1d', 'b200w_dtcwt_fwd_j1',
               'b200w_dtcwt_fwd_j2plus', 'b200w_dtcwt_inv_j1', 'b200w_dtcwt_inv_j2plus', 'b200w_scat_j1']
SYMBOLS = SYMBOLS + [s + '_generic' for s in KERNEL_ENTRIES] + [s + '_f64' for s in F64_ENTRIES] + [
    'b200w_dwt_forward_workspace', 'b200w_dwt_afb1d', 'b200w_dwt_sfb1d', 'b200w_comm_unique_id', 'b200w_comm_init', 'b200w_comm_destroy', 'b200w_allgather',
    'b200w_comm_last_error',
    'b200w_dtcwt_filter', 'b200w_dtcwt_dfilt', 'b200w_dtcwt_ifilt', 'b200w_dtcwt_filter_f64', 'b200w_dtcwt_dfilt_f64',
    'b200w_dtcwt_ifilt_f64']


class B200WaveError(RuntimeError):
    pass


def lib():
    """Load libb200wave.so (once).  Raises loudly when it is missing -- no CPU / eager fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise B200WaveError(
                'libb200wave.so is not built (%s). Build it with `python -m pytorch_wavelets_b200._build` '
                '(needs nvcc; compiles for sm_90a). There is no CPU fallback.' % SO_PATH)
        L = ctypes.CDLL(SO_PATH)
        L.b200w_strerror.restype = ctypes.c_char_p
        L.b200w_last_cuda_error.restype = ctypes.c_char_p
        pf = ctypes.c_void_p  # host tap pointers
        L.b200w_dwt_afb2d.argtypes = [c_vp, c_ll, c_int, c_vp, c_ll, c_int, c_vp, c_int, c_int, c_int,
                                      pf, pf, c_int, pf, pf, c_int, c_int, c_vp]
        L.b200w_dwt_sfb2d.argtypes = [c_vp, c_ll, c_int, c_vp, c_vp, c_ll, c_int, c_int, c_int, c_int, c_int, c_int,
                                      pf, pf, c_int, pf, pf, c_int, c_int, c_vp]
        hs = ctypes.POINTER(c_ll)
        L.b200w_dtcwt_fwd_j1.argtypes = [c_vp, c_ll, c_int, c_vp, c_ll, c_int, c_vp, hs, c_int, c_int, c_int, c_int,
                                         pf, c_int, pf, c_int, c_int, c_vp]
        L.b200w_dtcwt_fwd_j2plus.argtypes = [c_vp, c_ll, c_int, c_vp, c_ll, c_int, c_vp, hs, c_int, c_int, c_int,
                                             c_int, pf, pf, pf, pf, c_int, c_vp]
        L.b200w_dtcwt_inv_j1.argtypes = [c_vp, c_ll, c_int, c_vp, hs, c_vp, c_ll, c_int, c_int, c_int, c_int, c_int,
                                         pf, c_int, pf, c_int, c_int, c_vp]
        L.b200w_dtcwt_inv_j2plus.argtypes = [c_vp, c_ll, c_int, c_vp, hs, c_vp, c_ll, c_int, c_int, c_int, c_int,
                                             c_int, pf, pf, pf, pf, c_int, c_vp]
        L.b200w_scat_j1.argtypes = [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, pf, c_int, pf, c_int, c_int,
                                    ctypes.c_float, c_vp]
        L.b200w_dwt_forward.argtypes = [c_vp, c_ll, c_int, c_int, c_int, c_int, c_int, c_vp, ctypes.POINTER(c_vp),
                                        pf, pf, c_int, pf, pf, c_int, c_int, c_vp, c_ll, c_vp]
        L.b200w_dwt_forward_workspace.argtypes = [c_vp, c_ll, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int]
        L.b200w_dwt_forward_workspace.restype = c_ll
        L.b200w_dwt_afb1d.argtypes = [c_vp, c_ll, c_int, c_int, c_vp, c_vp, pf, pf, c_int, c_int, c_vp]
        L.b200w_dwt_sfb1d.argtypes = [c_vp, c_vp, c_int, c_int, c_vp, c_int, pf, pf, c_int, c_int, c_vp]
        L.b200w_comm_unique_id.argtypes = [c_vp]
        L.b200w_comm_init.argtypes = [ctypes.POINTER(c_vp), c_int, c_int, c_vp]
        L.b200w_comm_destroy.argtypes = [c_vp]
        L.b200w_allgather.argtypes = [c_vp, c_vp, c_vp, c_ll, c_vp]
        L.b200w_comm_last_error.restype = ctypes.c_char_p
        if hasattr(L, 'b200w_dtcwt_filter'):
            for sfx in ('', '_f64'):
                getattr(L, 'b200w_dtcwt_filter' + sfx).argtypes = [c_vp, c_vp, c_int, c_int, c_int, pf, c_int, c_int, c_int, c_vp]
                getattr(L, 'b200w_dtcwt_dfilt' + sfx).argtypes = [c_vp, c_vp, c_int, c_int, c_int, pf, pf, c_int, c_int, c_int, c_vp]
                getattr(L, 'b200w_dtcwt_ifilt' + sfx).argtypes = [c_vp, c_vp, c_int, c_int, c_int, pf, pf, c_int, c_int, c_int, c_vp]
        for s in KERNEL_ENTRIES:
            getattr(L, s + '_generic').argtypes = getattr(L, s).argtypes
        for s in F64_ENTRIES:
            if hasattr(L, s + '_f64'):   # (older experimental builds loaded through B200W_LIB lack them)
                getattr(L, s + '_f64').argtypes = [ctypes.c_double if a is ctypes.c_float else a
                                                   for a in getattr(L, s).argtypes]
        _lib = L
    return _lib


# Which implementation the launch wrappers call: the auto-selecting entry points, or (inside
# ``with generic_kernels():``, used by the A/B parity tests) the *_generic ones.  This switch lives in the Python
# shell; the C library itself has no global state.
_USE_GENERIC = False


class generic_kernels(object):
    def __enter__(self):
        global _USE_GENERIC
        self.prev, _USE_GENERIC = _USE_GENERIC, True
        return self

    def __exit__(self, *exc):
        global _USE_GENERIC
        _USE_GENERIC = self.prev
        return False


def entry(name, dtype=torch.float32):
    """The C-ABI function for a kernel entry point (honours ``generic_kernels``); float64 tensors take the ``_f64``
    entry points (generic tile kernels compiled for double -- the fast paths are float32-only)."""
    if dtype == torch.float64:
        return getattr(lib(), name + '_f64')
    return getattr(lib(), name + '_generic' if _USE_GENERIC else name)


def check(rc, what):
    """Map a negative return code to the exception type the reference raises in the same situation."""
    if rc == 0:
        return
    L = lib()
    msg = L.b200w_strerror(rc).decode()
    if rc == -1:
        raise ValueError('Unkown pad type')  # (sic) reference dwt/lowlevel.py:88,170,269
    if rc == -2:
        raise ValueError('%s: %s' % (what, msg))
    if rc == -6:
        raise NotImplementedError(what)
    if rc == -5:
        raise B200WaveError('%s: CUDA error: %s' % (what, L.b200w_last_cuda_error().decode()))
    raise B200WaveError('%s: %s (code %d)' % (what, msg, rc))


# ---- filter taps: host copies of the module buffers ------------------------------------------------
# Kernels take their taps as by-value parameters (constant bank), so the C ABI wants HOST arrays.
# Module buffers live on the device after .cuda(); reading them back costs a sync, so the host copy is
# cached ON THE TENSOR OBJECT together with its version counter: an in-place update (load_state_dict,
# .copy_()) invalidates it, and a new tensor that happens to reuse a freed address can never alias it.

class HostTaps(object):
    __slots__ = ('arr', 'ptr', 'n', 'arr64', 'ptr64')

    def __init__(self, arr):
        self.arr64 = np.ascontiguousarray(arr, dtype=np.float64).ravel()
        self.ptr64 = self.arr64.ctypes.data_as(ctypes.c_void_p)
        self.arr = np.ascontiguousarray(self.arr64, dtype=np.float32)
        self.ptr = self.arr.ctypes.data_as(ctypes.c_void_p)
        self.n = int(self.arr.size)

    def p(self, dtype):
        """Host pointer of the taps in the precision of the tensors of this call."""
        return self.ptr64 if dtype == torch.float64 else self.ptr


def host_taps(t):
    if isinstance(t, HostTaps):
        return t
    if not isinstance(t, torch.Tensor):
        return HostTaps(np.asarray(t, dtype=np.float64))
    # key: the version counter (in-place ops, optimiser steps, load_state_dict) AND the storage address
    # (`p.data = new_tensor` rebinding).  In-place edits made THROUGH `.data` (`p.data.mul_(2)`) bump neither:
    # call invalidate_host_taps(module_or_tensor) after such an edit.
    key = (t._version, t.data_ptr())
    cached = getattr(t, '_b200w_host_taps', None)
    if cached is not None and cached[0] == key:
        return cached[1]
    h = HostTaps(t.detach().to('cpu', torch.float64).numpy())
    try:
        t._b200w_host_taps = (key, h)
    except Exception:
        pass
    return h


def invalidate_host_taps(obj):
    """Drop the cached host copies of filter taps of a tensor, or of every parameter / buffer of a module
    (needed only after editing filters in place through ``.data``, which no version counter sees)."""
    ts = [obj] if isinstance(obj, torch.Tensor) else list(obj.parameters()) + list(obj.buffers())
    for t in ts:
        if hasattr(t, '_b200w_host_taps'):
            try:
                del t._b200w_host_taps
            except Exception:
                t._b200w_host_taps = None


# ---- tensors ------------------------------------------------------------------------------------------

def require_cuda_real(t, name, like=None):
    """CUDA float32 (every fast path) or float64 (generic kernels) tensors only; ``like``: dtype it must share."""
    if not isinstance(t, torch.Tensor):
        raise TypeError('%s must be a torch.Tensor' % name)
    if not t.is_cuda:
        raise NotImplementedError(
            '%s is on %s: the b200wave engine runs on CUDA (sm_90a) only and has no CPU fallback' % (name, t.device))
    if t.dtype not in (torch.float32, torch.float64):
        raise NotImplementedError('%s has dtype %s: the b200wave engine computes in float32 or float64' % (name, t.dtype))
    if like is not None and t.dtype != like:
        raise TypeError('%s has dtype %s, expected %s' % (name, t.dtype, like))   # the reference's conv2d raises too
    return t.dtype


require_cuda_f32 = require_cuda_real   # older name


def planes_view(t):
    """(tensor, plane_stride, pitch) for a 4-D (N,C,H,W) tensor whose (N,C) dims collapse to one plane
    index and whose rows are unit-stride; copies to contiguous only when the layout does not allow it."""
    N, C, H, W = t.shape
    s = t.stride()
    ok = (W == 1 or s[3] == 1) and s[2] >= W
    if ok and N > 1 and C > 1:
        ok = (s[0] == C * s[1])
    if not ok or t.numel() == 0:
        t = t.contiguous()
        s = t.stride()
    if C > 1:
        ps = s[1]
    elif N > 1:
        ps = s[0]
    else:
        ps = H * s[2]
    return t, int(ps), int(s[2])


def stream_of(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def hs_array(hs):
    return (c_ll * 6)(*[int(v) for v in hs])


# ---- optional per-call timing (bench.py roofline): CUDA events around each C-ABI launch ----------------
_RECORDER = None


class CallRecorder(object):
    """``with CallRecorder() as rec:`` brackets every kernel launch made through this module with CUDA
    events on the launching stream and remembers the algorithmic bytes (input read once + outputs written
    once) of that launch.  ``summary()`` synchronises and returns per-kernel averages."""

    def __init__(self):
        self.spans = []
        self.count = 0

    def __enter__(self):
        global _RECORDER
        _RECORDER = self
        return self

    def __exit__(self, *exc):
        global _RECORDER
        _RECORDER = None
        return False

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for tag, nbytes, e0, e1 in self.spans:
            d = out.setdefault(tag, {'tag': tag, 'count': 0, 'total_ms': 0.0, 'alg_bytes': nbytes})
            d['count'] += 1
            d['total_ms'] += e0.elapsed_time(e1)
        for d in out.values():
            d['avg_ms'] = d['total_ms'] / d['count']
        return out


class span(object):
    """Context manager used by the launch wrappers; free when no recorder is active."""
    __slots__ = ('tag', 'nbytes', 'e0', 'rec')

    def __init__(self, tag, nbytes):
        self.tag, self.nbytes, self.rec = tag, nbytes, _RECORDER

    def __enter__(self):
        if self.rec is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.rec is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            self.rec.spans.append((self.tag() if callable(self.tag) else self.tag, self.nbytes, self.e0, e1))
            self.rec.count += 1
        return False
