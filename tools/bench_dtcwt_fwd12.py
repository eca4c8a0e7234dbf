"""Time DTCWT forward levels 1 + 2 in one call (FWD_J12's fwd_j12) against the per-level composition on one GPU.

    python tools/bench_dtcwt_fwd12.py --out DIR [--iters 20] [--warmup 3]

The per-level route is ``fwd_j1`` followed by ``fwd_j2plus`` on its low-pass (the level functions, called directly: the
full-resolution level-1 low-pass goes to HBM and back); the fused route is ``fwd_j12``, which runs one kernel where its
plan accepts the shape and the same two level kernels otherwise.  near_sym_a / qshift_a, symmetric, float32, about
0.8 GB of input per shape.  The routes alternate call by call (CUDA events around each call, after warm-up); the report
gives the median and the spread (max - min) of each route, the ratio of the medians, the algorithmic bytes of the fused
route (x + LL2 + yh0 + yh1) and their rate, and the card name, power limit and SM clock read in the same run.  The two
routes' outputs must be equal bit for bit.  Writes DIR/bench_dtcwt_fwd12.json.
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
from pytorch_wavelets_b200 import _ffi  # noqa: E402
from pytorch_wavelets_b200.dtcwt import transform_funcs as tf  # noqa: E402

# the bench shape, three narrower plane classes, and one the plan rejects (wider than the fused CTA holds)
SHAPES = [(64, 3, 1024, 1024), (256, 3, 512, 512), (1024, 3, 256, 256), (4096, 3, 128, 128), (16, 3, 2048, 2048)]


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(','), [v.strip() for v in out.split(',')]))
    except Exception as e:   # (report what failed; the timings stand on their own)
        return {'error': repr(e), 'name': torch.cuda.get_device_name()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    m = pw.DTCWTForward(biort='near_sym_a', qshift='qshift_a').cuda()
    taps = [_ffi.host_taps(getattr(m, k)) for k in ('h0o', 'h1o', 'h0a', 'h1a', 'h0b', 'h1b')]
    o5, ri = tf.get_dimensions5(2, -1)[:2]

    def per_level(x):
        ll1, h0 = tf.fwd_j1(x, taps[0], taps[1], False, o5, ri, 1)
        ll2, h1 = tf.fwd_j2plus(ll1, *taps[2:], False, o5, ri)
        return ll2, h0, h1

    def fused(x):
        return tf.fwd_j12(x, *taps, False, o5, ri, 1)

    rows = []
    info = gpu_info()
    with torch.no_grad():
        for shape in SHAPES:
            N, C, H, W = shape
            x = torch.randn(shape, device='cuda')
            a, b = per_level(x), fused(x)
            equal = all(torch.equal(u, v) for u, v in zip(a, b))
            del a, b
            route = 'fused' if _ffi.lib().b200w_dtcwt_fwd_j12_workspace(
                x.data_ptr(), H * W, W, 16, N, C, H, W, taps[0].n, taps[1].n, taps[2].n) == 0 else 'levels'
            for _ in range(args.warmup):
                per_level(x)
                fused(x)
            t = {'levels': [], 'fused': []}
            for _ in range(args.iters):
                for name, fn in (('levels', per_level), ('fused', fused)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn(x)
                    e1.record()
                    e1.synchronize()
                    t[name].append(e0.elapsed_time(e1))
            med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
            spread = {k: max(v) - min(v) for k, v in t.items()}
            alg = 4.0 * N * C * H * W * 5
            rows.append({'shape': list(shape), 'fused_route': route, 'bit_equal': equal,
                         'levels_ms': round(med['levels'], 4), 'levels_spread_ms': round(spread['levels'], 4),
                         'fused_ms': round(med['fused'], 4), 'fused_spread_ms': round(spread['fused'], 4),
                         'ratio': round(med['fused'] / med['levels'], 4), 'alg_bytes': alg,
                         'fused_TBps': round(alg / med['fused'] / 1e9, 3)})
            print(json.dumps(rows[-1]), flush=True)
            del x
            torch.cuda.empty_cache()
    res = {'gpu': info, 'gpu_after': gpu_info(), 'iters': args.iters, 'rows': rows}
    with open(os.path.join(args.out, 'bench_dtcwt_fwd12.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res['gpu']))
    if not all(r['bit_equal'] for r in rows):
        sys.exit('the fused and per-level routes differ')


if __name__ == '__main__':
    main()
