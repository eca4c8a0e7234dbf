"""CPU: libb200wave.so builds/loads and exports every symbol include/b200wave.h declares; host-side
helpers (no compute, no GPU)."""
import ctypes
import os
import re

import pytest

from pytorch_wavelets_b200 import _build, _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _ffi.lib()


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, 'include', 'b200wave.h')).read()
    declared = sorted(set(re.findall(r'\b(b200w_[a-z0-9_]+)\s*\(', hdr)))
    assert declared, 'no declarations found'
    for name in declared:
        assert hasattr(lib, name), 'libb200wave.so does not export %s' % name
    assert sorted(_ffi.SYMBOLS) == declared


def test_version_and_strerror(lib):
    assert lib.b200w_version() == 100
    assert lib.b200w_strerror(0) == b'ok'
    assert lib.b200w_strerror(-1) == b'Unkown pad type'
    assert lib.b200w_last_cuda_error() == b''


def test_length_rules(lib):
    # pywt.dwt_coeff_len / reference dwt/lowlevel.py:153 and :242-267
    assert lib.b200w_dwt_coeff_len(512, 8, 1) == 259
    assert lib.b200w_dwt_coeff_len(259, 8, 1) == 133
    assert lib.b200w_dwt_coeff_len(133, 8, 0) == 70
    assert lib.b200w_dwt_coeff_len(127, 8, 2) == 64
    assert lib.b200w_dwt_coeff_len(2048, 16, 0) == 1031
    assert lib.b200w_dwt_rec_len(259, 8, 1) == 512
    assert lib.b200w_dwt_rec_len(64, 8, 2) == 128
    assert lib.b200w_dwt_coeff_len(0, 8, 1) < 0


def test_argument_validation_without_gpu(lib):
    """Validation happens before any CUDA call, so bad arguments are reported on a CPU-only box."""
    f = (ctypes.c_float * 8)(*([0.5] * 8))
    fp = ctypes.cast(f, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    rc = lib.b200w_dwt_afb2d(buf, 64, 8, buf, 49, 7, buf, 1, 8, 8, fp, fp, 8, fp, fp, 8, 3, None)
    assert rc == -1  # 'constant' is not a filter-bank mode (reference ValueError)
    rc = lib.b200w_dwt_afb2d(buf, 64, 8, buf, 49, 7, buf, 1, 8, 8, fp, fp, 8, fp, fp, 8, 99, None)
    assert rc == -1
    rc = lib.b200w_dwt_afb2d(None, 64, 8, buf, 49, 7, buf, 1, 8, 8, fp, fp, 8, fp, fp, 8, 1, None)
    assert rc == -3
    hs = (ctypes.c_longlong * 6)(1, 1, 1, 1, 1, 1)
    rc = lib.b200w_dtcwt_fwd_j2plus(buf, 36, 6, buf, 9, 3, buf, hs, 1, 1, 6, 6, fp, fp, fp, fp, 8, None)
    assert rc == -2  # rows/cols must be a multiple of 4 (reference ValueError)
    rc = lib.b200w_dtcwt_fwd_j1(buf, 64, 8, buf, 64, 8, buf, hs, 1, 1, 8, 8, fp, 8, fp, 7, 1, None)
    assert rc == -4  # even-length level-1 filter


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_ffi, '_lib', None)
    monkeypatch.setattr(_ffi, 'SO_PATH', str(tmp_path / 'nope.so'))
    with pytest.raises(_ffi.B200WaveError):
        _ffi.lib()


def test_f64_and_primitive_entries_validate_without_gpu(lib):
    """The float64 and standalone-primitive entry points share the validation of the float32 ones (launch_params.h is a
    template on the element type; csrc/k_prims.cu checks sizes before launching)."""
    d = (ctypes.c_double * 10)(*([0.25] * 10))
    dp = ctypes.cast(d, ctypes.c_void_p)
    buf = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    assert lib.b200w_dwt_afb2d_f64(buf, 64, 8, buf, 49, 7, buf, 1, 8, 8, dp, dp, 8, dp, dp, 8, 99, None) == -1   # bad mode
    assert lib.b200w_dwt_afb2d_f64(None, 64, 8, buf, 49, 7, buf, 1, 8, 8, dp, dp, 8, dp, dp, 8, 1, None) == -3  # null input
    hs = (ctypes.c_longlong * 6)(1, 1, 1, 1, 1, 1)
    assert lib.b200w_dtcwt_fwd_j2plus_f64(buf, 36, 6, buf, 9, 3, buf, hs, 1, 1, 6, 6, dp, dp, dp, dp, 8, None) == -2
    f = (ctypes.c_float * 10)(*([0.25] * 10))
    fp = ctypes.cast(f, ctypes.c_void_p)
    # coldfilt needs rows % 4 == 0, colifilt rows % 2 == 0 (reference ValueError), q-shift filters an even length
    assert lib.b200w_dtcwt_dfilt(buf, buf, 1, 18, 16, fp, fp, 10, 0, 0, None) == -2
    assert lib.b200w_dtcwt_dfilt(buf, buf, 1, 16, 18, fp, fp, 10, 0, 1, None) == -2
    assert lib.b200w_dtcwt_ifilt(buf, buf, 1, 15, 16, fp, fp, 10, 0, 0, None) == -2
    assert lib.b200w_dtcwt_dfilt(buf, buf, 1, 16, 16, fp, fp, 9, 0, 0, None) == -4
    assert lib.b200w_dtcwt_filter(None, buf, 1, 16, 16, fp, 4, 1, 0, None) == -3
    assert lib.b200w_dtcwt_filter(buf, buf, 1, 16, 16, fp, 41, 1, 0, None) == -4       # longer than B200W_MAX_TAPS
    # empty batches are a no-op everywhere (no launch, no CUDA call)
    assert lib.b200w_dtcwt_filter(buf, buf, 0, 16, 16, fp, 4, 1, 0, None) == 0
    assert lib.b200w_dtcwt_filter_f64(buf, buf, 0, 16, 16, dp, 5, 0, 1, None) == 0


def test_shells_refuse_cpu_tensors_and_unsupported_dtypes():
    """No CPU or eager fallback anywhere: CPU tensors and dtypes other than float32 / float64 raise."""
    import torch
    import pytorch_wavelets_b200 as pw
    from pytorch_wavelets_b200.dtcwt import lowlevel as ll
    x = torch.randn(1, 1, 16, 16)
    for mod in (pw.DWTForward(J=1, wave='bior2.2'), pw.DTCWTForward(J=1), pw.ScatLayer()):
        with pytest.raises(NotImplementedError):
            mod(x)
        with pytest.raises(NotImplementedError):
            mod.double()(x.double())
    with pytest.raises(NotImplementedError):
        ll.colfilter(x, torch.ones(4))
    with pytest.raises(NotImplementedError):
        ll.coldfilt(x, torch.ones(10), torch.ones(10))
    with pytest.raises(NotImplementedError):
        _ffi.require_cuda_real(torch.zeros(2, dtype=torch.float16), 'x')
