"""Time the 1-D scattering layers (ScatLayer1D / ScatLayer1Dj2) against the composition they replace, on one GPU.

    python tools/bench_scat1d.py --out DIR [--iters 20] [--warmup 3]

Workloads: the two 1 GiB float32 inputs of tools/bench_dtcwt1d.py, long rows (64, 16, 262144) and many short rows
(4096, 64, 1024); near_sym_a / qshift_a, symmetric mode, magbias 1e-2.  Legs: j1 and j2, each as a forward without a
gradient and as a forward with a gradient plus the backward pass.  The other route is what a user composed before: the
differentiable 1-D level Functions (``FWD1D_J1`` / ``FWD1D_J2PLUS``, one kernel per level), ``F.avg_pool1d``, the
smoothed magnitude as torch pointwise ops and ``torch.cat``, with autograd's backward.  The routes alternate call by
call (CUDA events around each call, after warm-up).  The forward outputs of both routes must be equal at the timed
sizes.  The report gives medians and the range of the timed calls, the card name and power limit read in the same run,
and the algorithmic bytes of the fused route over the 3.35 TB/s data-sheet HBM3 bandwidth.  Algorithmic bytes count
every tensor a launch must read or write once (float32, per input sample): j1 forward 8 B (x in; pooled low-pass and
magnitude out), 12 B with the derivatives; j2 forward 20 B (three launches through the level-1 low-pass and magnitude
workspaces), 28 B with the derivatives; the backward passes read the output gradient and the derivatives and write the
input gradient once: 12 B (j1) and 16 B (j2).  Writes DIR/bench_scat1d.json.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pytorch_wavelets_b200 as pw  # noqa: E402
from pytorch_wavelets_b200.dtcwt import transform1d as t1  # noqa: E402
from tools.bench_dtcwt1d import HBM_BYTES_PER_S, SHAPES, gpu_info, time_pair  # noqa: E402

BIAS = 1e-2
# algorithmic bytes per float32 input sample: (forward without derivatives, forward with derivatives + backward)
BYTES_PER_SAMPLE = {'j1': (8, 12 + 12), 'j2': (20, 28 + 16)}


def _mag(yh):
    return torch.sqrt(yh[..., 0] ** 2 + yh[..., 1] ** 2 + BIAS ** 2) - BIAS


def composed_j1(m, x):
    lo, yh = t1.FWD1D_J1.apply(x, m.h0o, m.h1o, False, 1)
    return torch.cat((F.avg_pool1d(lo, 2), _mag(yh)), dim=1)


def composed_j2(m, x):
    lo1, yh1 = t1.FWD1D_J1.apply(x, m.h0o, m.h1o, False, 1)
    lo2, yh2 = t1.FWD1D_J2PLUS.apply(lo1, m.h0a, m.h1a, m.h0b, m.h1b, False)
    u, yhu = t1.FWD1D_J1.apply(_mag(yh1), m.h0o, m.h1o, False, 1)
    return torch.cat((F.avg_pool1d(lo2, 2), F.avg_pool1d(u, 2), _mag(yh2), _mag(yhu)), dim=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    dev = 'cuda:0'
    rows = []
    info = gpu_info()
    layers = {'j1': (pw.ScatLayer1D().to(dev), composed_j1), 'j2': (pw.ScatLayer1Dj2().to(dev), composed_j2)}
    for sname, shape in SHAPES.items():
        x = torch.randn(shape, device=dev)
        xg = x.clone().requires_grad_(True)
        for leg, (m, composed) in layers.items():
            z = m(x)
            assert torch.equal(z, composed(m, x)), 'forward routes differ'
            dz = torch.randn_like(z)
            del z

            def fused_grad():
                torch.autograd.grad(m(xg), (xg,), dz)

            def composed_grad():
                torch.autograd.grad(composed(m, xg), (xg,), dz)

            for grad, fa, fb in ((False, lambda: m(x), lambda: composed(m, x)), (True, fused_grad, composed_grad)):
                ma, mb, sa, sb = time_pair(fa, fb, a.iters, a.warmup)
                nb = shape[0] * shape[1] * shape[2] * BYTES_PER_SAMPLE[leg][grad]
                rows.append({'workload': sname, 'shape': list(shape), 'layer': leg,
                             'pass': 'forward+backward' if grad else 'forward', 'fused_ms': ma, 'composed_ms': mb,
                             'fused_range_ms': sa, 'composed_range_ms': sb, 'speedup': mb / ma, 'alg_bytes': nb,
                             'hbm_fraction': nb / (ma * 1e-3) / HBM_BYTES_PER_S})
                print(json.dumps(rows[-1]))
            del dz
            torch.cuda.empty_cache()
        del x, xg
        torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_scat1d.json'), 'w') as fh:
        json.dump({'gpu': info, 'iters': a.iters, 'rows': rows}, fh, indent=1)
    print(json.dumps({'gpu': info}))


if __name__ == '__main__':
    main()
