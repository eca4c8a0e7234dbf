"""Time the 1-D DTCWT level kernels against the composition of the standalone GPU primitives on one GPU.

    python tools/bench_dtcwt1d.py --out DIR [--iters 20] [--warmup 3]

Workloads: DTCWT1DForward / DTCWT1DInverse, near_sym_a / qshift_a, J = 1 and J = 4, symmetric mode, float32, on long
rows (64, 16, 262144) and on many short rows (4096, 64, 1024), 1 GiB each.  The other route is what the package offered
before: per level ``dtcwt.lowlevel.rowfilter`` / ``rowdfilt`` / ``rowifilt`` on (N, C, 1, n) views plus a torch add for
the inverse.  The routes alternate call by call (CUDA events around each call, after warm-up); the report gives the
median of the timed calls, the algorithmic bytes (every level's input read once and outputs written once) and their
fraction of the 3.35 TB/s data-sheet HBM3 bandwidth, and the card name and power limit read in the same run.  At the
timed sizes the two routes' outputs must be equal.  Writes DIR/bench_dtcwt1d.json.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pytorch_wavelets_b200 as pw  # noqa: E402
from pytorch_wavelets_b200.dtcwt import lowlevel as ll  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = {'long': (64, 16, 262144), 'short': (4096, 64, 1024)}


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(','), [v.strip() for v in out.split(',')]))
    except Exception as e:   # (report what failed; the timings stand on their own)
        return {'error': repr(e), 'name': torch.cuda.get_device_name()}


def prim_forward(f, x, J):
    """The forward through the standalone primitives; same outputs as DTCWT1DForward."""
    x4 = x[:, :, None, :]
    lo, hi = ll.rowfilter(x4, f.h0o), ll.rowfilter(x4, f.h1o)
    yh = [hi.view(x.shape[0], x.shape[1], -1, 2)]
    for _ in range(1, J):
        assert lo.shape[-1] % 4 == 0
        hi = ll.rowdfilt(lo, f.h1b, f.h1a, highpass=True)
        lo = ll.rowdfilt(lo, f.h0b, f.h0a)
        yh.append(hi.view(x.shape[0], x.shape[1], -1, 2))
    return lo[:, :, 0], yh


def prim_inverse(i, yl, yh):
    lo = yl[:, :, None, :]
    N, C = yl.shape[:2]
    for j in range(len(yh) - 1, 0, -1):
        lo = ll.rowifilt(lo, i.g0b, i.g0a) + ll.rowifilt(yh[j].reshape(N, C, 1, -1), i.g1b, i.g1a, highpass=True)
    y = ll.rowfilter(lo, i.g0o) + ll.rowfilter(yh[0].reshape(N, C, 1, -1), i.g1o)
    return y[:, :, 0]


def alg_bytes(shape, J, inverse):
    """Every level reads its input once and writes its outputs once (float32)."""
    N, C, n = shape
    total = 3 * n                       # level 1: x in, lo and hi out (and the reverse)
    k = n
    for _ in range(1, J):
        total += 2 * k                  # j >= 2: k in, k/2 + k/2 out (inverse: k/2 + k/2 in, k out)
        k //= 2
    return 4 * N * C * total


def time_pair(fa, fb, iters, warmup):
    for _ in range(warmup):
        fa()
        fb()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(iters):
        for f, t in ((fa, ta), (fb, tb)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            t.append(e0.elapsed_time(e1))
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    return med(ta), med(tb), (min(ta), max(ta)), (min(tb), max(tb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    dev = 'cuda:0'
    rows = []
    info = gpu_info()
    for sname, shape in SHAPES.items():
        x = torch.randn(shape, device=dev)
        for J in (1, 4):
            f = pw.DTCWT1DForward(J=J).to(dev)
            i = pw.DTCWT1DInverse().to(dev)
            yl, yh = f(x)
            pyl, pyh = prim_forward(f, x, J)
            assert torch.equal(yl, pyl) and all(torch.equal(u, v) for u, v in zip(yh, pyh)), 'forward routes differ'
            assert torch.equal(i((yl, yh)), prim_inverse(i, yl, yh)), 'inverse routes differ'
            del pyl, pyh
            for direction, fa, fb in (('forward', lambda: f(x), lambda: prim_forward(f, x, J)),
                                      ('inverse', lambda: i((yl, yh)), lambda: prim_inverse(i, yl, yh))):
                ma, mb, sa, sb = time_pair(fa, fb, a.iters, a.warmup)
                nb = alg_bytes(shape, J, direction == 'inverse')
                rows.append({'workload': sname, 'shape': list(shape), 'J': J, 'direction': direction,
                             'kernels_ms': ma, 'primitives_ms': mb, 'kernels_range_ms': sa, 'primitives_range_ms': sb,
                             'speedup': mb / ma, 'alg_bytes': nb, 'hbm_fraction': nb / (ma * 1e-3) / HBM_BYTES_PER_S})
                print(json.dumps(rows[-1]))
            del yl, yh
            torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_dtcwt1d.json'), 'w') as fh:
        json.dump({'gpu': info, 'iters': a.iters, 'rows': rows}, fh, indent=1)
    print(json.dumps({'gpu': info}))


if __name__ == '__main__':
    main()
