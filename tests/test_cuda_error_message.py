"""CPU: a failed launch of a float64 kernel, a 1-D kernel or a DTCWT primitive reports its own CUDA error through
b200w_last_cuda_error(), not an empty string or the message of an earlier call.  On a machine without a usable GPU every
launch fails, so valid arguments give B200W_ECUDA and the error text of that launch."""
import subprocess
import sys

import pytest
import torch

from pytorch_wavelets_b200 import _build

# Runs in a fresh process, so the error buffer starts empty.  Filter taps are real host arrays (the library copies them
# into the kernel parameters); the device pointers are placeholders, never dereferenced because no launch succeeds.
_SCRIPT = r'''
import ctypes, sys
lib = ctypes.CDLL(sys.argv[1])
lib.b200w_last_cuda_error.restype = ctypes.c_char_p
P = ctypes.c_void_p(4096)
LL = ctypes.c_longlong
d2 = (ctypes.c_double * 2)(0.5, 0.5)
f2 = (ctypes.c_float * 2)(0.5, 0.5)
d3 = (ctypes.c_double * 3)(0.25, 0.5, 0.25)
calls = {
    'b200w_dwt_afb2d_f64': lambda: lib.b200w_dwt_afb2d_f64(P, LL(256), 16, P, LL(64), 8, P, 1, 16, 16, d2, d2, 2, d2,
                                                          d2, 2, 1, None),
    'b200w_dwt_afb1d': lambda: lib.b200w_dwt_afb1d(P, LL(32), 1, 32, P, P, f2, f2, 2, 1, None),
    'b200w_dtcwt_filter_f64': lambda: lib.b200w_dtcwt_filter_f64(P, P, 1, 8, 8, d3, 3, 1, 0, None),
}
for name, call in calls.items():
    print(name, call(), lib.b200w_last_cuda_error().decode())
'''


@pytest.mark.skipif(torch.cuda.is_available(), reason='launches with placeholder device pointers: CPU-only machines')
def test_failed_launch_records_its_cuda_error():
    so = _build.build()
    out = subprocess.run([sys.executable, '-c', _SCRIPT, so], capture_output=True, text=True, check=True).stdout
    lines = out.strip().splitlines()
    assert len(lines) == 3, out
    for line in lines:
        name, rc, msg = line.split(' ', 2)
        assert int(rc) == -5, line
        assert msg.startswith('cudaError'), line
