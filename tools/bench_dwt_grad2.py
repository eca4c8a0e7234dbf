"""Time the DWT's first- and second-order backward passes against the same graphs written as torch ops, on one GPU.

    python tools/bench_dwt_grad2.py --out DIR [--shape 128 32 512 512] [--r1-batch 32] [--iters 10] [--warmup 2]

DWTForward(J=3, 'db4', 'symmetric') / DWTInverse, float32 (the headline DWT shape of bench.py).  Legs:
  first_order  DWTForward forward + a plain .backward() at --shape (the route the package always took);
  r1_forward   one R1 step: logit = linear(features), loss = softplus(logit), penalty = |d loss / d x|^2,
               (loss + penalty).backward(), through DWTForward, batch --r1-batch of --shape (the torch-op graph of a
               full batch does not fit in 80 GB);
  r1_inverse   the same with DWTInverse between the coefficients and the linear layer;
  adjoint      the transposed analysis (b200w_dwt_afb2d_adjoint) against the plain cropped synthesis level
               (sfb2d_level) on the level-1 coefficients of --shape: one border kernel more.
The torch-op routes are tests/test_gpu_dwt_grad2.py's restatement (extension gather + strided conv2d /
conv_transpose2d, TF32 off); tests/test_gpu_dwt_grad2.py checks that both give the same gradients (in float64:
the R1 weight gradient is too badly conditioned to compare in float32).  Routes alternate call by call, CUDA events around each call after warm-up; medians and ranges are
reported.  Algorithmic bytes: one transform pass reads its input and writes its output once (float32): the image and
all coefficient bands.  first_order is 2 passes, an R1 step 4 (forward, its backward, and that backward's transpose
and backward again), the adjoint / synthesis level 4 Hc Wc + H W floats per plane.  Also reports the card name and
power limit read in the same run.  Writes DIR/bench_dwt_grad2.json.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pytorch_wavelets_b200 as pw  # noqa: E402
from pytorch_wavelets_b200 import _ffi  # noqa: E402
from pytorch_wavelets_b200.dwt import lowlevel  # noqa: E402
from tests import test_gpu_dwt_grad2 as tg  # noqa: E402
from tools.bench_dtcwt1d import HBM_BYTES_PER_S, gpu_info, time_pair  # noqa: E402

MODE, WAVE, J = 'symmetric', 'db4', 3


def pass_bytes(shape):
    """Bytes of one transform pass: the image, every band-pass and the final low-pass, float32."""
    N, C, H, W = shape
    m, n, h, w = lowlevel.mode_to_int(MODE), H * W, H, W
    for _ in range(J):
        h, w = _ffi.lib().b200w_dwt_coeff_len(h, 8, m), _ffi.lib().b200w_dwt_coeff_len(w, 8, m)
        n += 3 * h * w
    return 4 * N * C * (n + h * w)


def leg(name, fa, fb, nbytes, iters, warmup):
    a, b, ra, rb = time_pair(fa, fb, iters, warmup)
    return dict(leg=name, ours_ms=a, torch_ops_ms=b, ours_range_ms=ra, torch_ops_range_ms=rb, speedup=b / a,
                algorithmic_bytes=nbytes, ours_bytes_per_s=nbytes / (a * 1e-3),
                ours_share_of_hbm_datasheet=nbytes / (a * 1e-3) / HBM_BYTES_PER_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--shape', type=int, nargs=4, default=[128, 32, 512, 512])
    ap.add_argument('--r1-batch', type=int, default=32)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_dwt_grad2 needs a CUDA device')
    dev = 'cuda:0'
    torch.backends.cudnn.allow_tf32 = False    # the torch-op graphs' convolutions in true float32, as ours
    torch.manual_seed(0)
    f = pw.DWTForward(J=J, wave=WAVE, mode=MODE).to(dev)
    i = pw.DWTInverse(wave=WAVE, mode=MODE).to(dev)
    h0, h1 = f.h0_col.flatten(), f.h1_col.flatten()
    g0, g1 = i.g0_col.flatten(), i.g1_col.flatten()
    res = dict(gpu=gpu_info(), shape=a.shape, r1_batch=a.r1_batch, wave=WAVE, mode=MODE, J=J, legs=[])

    # first-order: forward + plain backward
    x = torch.randn(*a.shape, device=dev, requires_grad=True)

    def fo(fwd):
        def run():
            yl, yh = fwd(x)
            torch.autograd.backward([yl] + yh, [torch.ones_like(yl)] + [torch.ones_like(h) for h in yh])
            x.grad = None
        return run
    res['legs'].append(leg('first_order', fo(f), fo(lambda x: tg.dwt_torch(x, h0, h1, MODE, J)),
                           2 * pass_bytes(a.shape), a.iters, a.warmup))
    del x
    torch.cuda.empty_cache()

    # R1 steps
    shape = [a.r1_batch] + a.shape[1:]
    xr = torch.randn(*shape, device=dev)
    for case in ('forward', 'inverse'):
        if case == 'forward':
            ours = lambda x: (lambda r: [r[0]] + r[1])(f(x))                                  # noqa: E731
            ops = lambda x: (lambda r: [r[0]] + r[1])(tg.dwt_torch(x, h0, h1, MODE, J))       # noqa: E731
            leaves = [xr]
        else:
            yl, yh = f(xr)
            ours = lambda *c: [i((c[0], list(c[1:])))]                                        # noqa: E731
            ops = lambda *c: [tg.idwt_torch(c[0], list(c[1:]), g0, g1, MODE)]                 # noqa: E731
            leaves = [yl] + yh
        nfeat = sum(t.numel() // t.shape[0] for t in ours(*leaves))
        lin = torch.nn.Linear(nfeat, 1).to(dev)
        torch.nn.init.normal_(lin.weight, std=nfeat ** -0.5)
        lv = [t.detach().clone().requires_grad_(True) for t in leaves]
        res['legs'].append(leg('r1_' + case, lambda: tg.r1_step(ours, lv, lin), lambda: tg.r1_step(ops, lv, lin),
                               4 * pass_bytes(shape), a.iters, a.warmup))
        del lin, lv
        torch.cuda.empty_cache()

    # the adjoint level against the plain cropped synthesis level
    N, C, H, W = a.shape
    m = lowlevel.mode_to_int(MODE)
    Hc, Wc = _ffi.lib().b200w_dwt_coeff_len(H, 8, m), _ffi.lib().b200w_dwt_coeff_len(W, 8, m)
    ll = torch.randn(N, C, Hc, Wc, device=dev)
    hs = torch.randn(N, C, 3, Hc, Wc, device=dev)
    taps = [_ffi.host_taps(t) for t in (f.h0_row, f.h1_row, f.h0_col, f.h1_col)]
    r = leg('adjoint_vs_sfb2d', lambda: lowlevel.afb2d_adjoint_level(ll, hs, *taps, m, (H, W)),
            lambda: lowlevel.sfb2d_level(ll, hs, *taps, m, out_hw=(H, W)),
            4 * N * C * (4 * Hc * Wc + H * W), a.iters, a.warmup)
    r['note'] = 'torch_ops_* here is the plain synthesis level sfb2d_level (the first-order backward of AFB2D)'
    res['legs'].append(r)

    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_dwt_grad2.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
