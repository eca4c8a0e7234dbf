"""Time the 2-D wavelet packet transform (WPT2DForward / WPT2DInverse) against the composition a user builds without
it, on one GPU.

    python tools/bench_wpt2d.py --out DIR [--iters 10] [--warmup 3]

Workload: (64, 3, 1024, 1024) float32 (768 MiB), J = 1, 3 and 5, db4 and haar, periodization and symmetric.  J = 5 ends
at 32 x 32 planes (haar, periodization) or 38 x 38 (db4 symmetric), the small-plane regime of a packet tree.  The other
route is the
hand-built composition: ``DWTForward(J=1)`` on all nodes of a level and ``torch.cat`` of its low-pass and band-pass
outputs into the next level's input; the inverse takes each group of four children apart, runs ``DWTInverse`` and
crops the result to the level's size.  The two routes alternate call by call (CUDA events around each call, after
warm-up); the report gives medians and the range of the timed calls.  At the timed sizes the two analysis outputs must
be equal and the two reconstructions within 1e-5 of max|x| of each other (the tests' perfect-reconstruction bound).
Algorithmic bytes: every level reads its input once and writes its output once (float32); their sum over the time is
compared with the 3.35 TB/s data-sheet HBM3 bandwidth.  A per-level breakdown (CUDA events around each level launch,
separate calls) names the route each level took.  The card name, power limit and SM clock are read in the same run.
The route probe then times one level on small planes (8 to 40 columns on the small side, about 768 MiB of input) on the
streaming kernel, as the packet level routes it, and on the tile kernel.  Writes DIR/bench_wpt2d.json.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pytorch_wavelets_b200 as pw  # noqa: E402
from pytorch_wavelets_b200 import _ffi, wavelets  # noqa: E402
from pytorch_wavelets_b200.dwt import packet2d  # noqa: E402
from tests.test_gpu_wpt2d import predicted_routes  # noqa: E402
from tools.bench_dtcwt1d import HBM_BYTES_PER_S, gpu_info, time_pair  # noqa: E402

SHAPE = (64, 3, 1024, 1024)
CONFIGS = [(J, wave, mode) for J in (1, 3, 5) for wave in ('db4', 'haar') for mode in ('periodization', 'symmetric')]


def composed_forward(x, fwd1, J):
    N, C = x.shape[:2]
    y = x
    for _ in range(J):
        B, P = y.shape[:2]
        yl, yh = fwd1(y)
        y = torch.cat([yl[:, :, None], yh[0]], 2).reshape(B, 4 * P, yl.shape[-2], yl.shape[-1])
    return y.reshape(N, C, 4 ** J, y.shape[-2], y.shape[-1])


def composed_inverse(y, inv, sizes):
    N, C, P = y.shape[:3]
    c = y.reshape(N, C * P, y.shape[3], y.shape[4])
    for h, w in sizes[-2::-1]:
        B, P4, Hc, Wc = c.shape
        q = c.reshape(B, P4 // 4, 4, Hc, Wc)
        c = inv((q[:, :, 0], [q[:, :, 1:]]))[..., :h, :w]
    return c


def time_routes(fns, iters, warmup):
    """Median and range (ms) of each function, called in turn (CUDA events around each call) after warm-up."""
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(iters):
        for f, t in zip(fns, ts):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            t.append(e0.elapsed_time(e1))
    return [(sorted(t)[len(t) // 2], min(t), max(t)) for t in ts]


def route_probe(dev, iters, warmup):
    """One level on small planes, about 768 MiB of float32 input per call: the streaming kernel (through the DWT level
    functions, the same kernel body), the packet level as csrc/wpt2d.cu routes it, and the tile kernel (the packet level
    under ``generic_kernels()``).  The db4 symmetric inputs have odd widths, so their analysis cannot stream."""
    rows = []
    for wave, mode in (('haar', 'periodization'), ('db4', 'symmetric')):
        L = len(wavelets.Wavelet(wave).dec_lo)
        m = pw.dwt.lowlevel.mode_to_int(mode)
        f = pw.DWTForward(wave=wave, mode=mode)
        an = [f.h0_col, f.h1_col, f.h0_row, f.h1_row]
        i = pw.DWTInverse(wave=wave, mode=mode)
        sy = [i.g0_col, i.g1_col, i.g0_row, i.g1_row]
        for wo in (8, 16, 32, 40):
            n = 2 * wo if mode == 'periodization' else 2 * wo - L + 1
            P = 1024 * 1024 // (n * n)
            x = torch.randn(SHAPE[0] * SHAPE[1], P, n, n, device=dev)
            c = torch.randn(SHAPE[0] * SHAPE[1], 4 * P, wo, wo, device=dev)
            ll = torch.randn(SHAPE[0] * SHAPE[1], P, wo, wo, device=dev)
            hi = torch.randn(SHAPE[0] * SHAPE[1], P, 3, wo, wo, device=dev)

            def generic(fn):
                def run():
                    with _ffi.generic_kernels():
                        fn()
                return run
            afb = lambda: packet2d.wpt_afb2d_level(x, *an, m)   # noqa: E731
            sfb = lambda: packet2d.wpt_sfb2d_level(c, *sy, m)   # noqa: E731
            res = time_routes([lambda: pw.dwt.lowlevel.afb2d_level(x, *an, m), afb, generic(afb),
                               lambda: pw.dwt.lowlevel.sfb2d_level(ll, hi, *sy, m), sfb, generic(sfb)], iters, warmup)
            ho = wo if mode == 'periodization' else 2 * wo - L + 2
            for k, (leg, route) in enumerate([('analysis', 'stream'), ('analysis', 'packet'), ('analysis', 'tile'),
                                              ('synthesis', 'stream'), ('synthesis', 'packet'),
                                              ('synthesis', 'tile')]):
                nb = 4 * x.shape[0] * P * ((n * n + 4 * wo * wo) if leg == 'analysis' else (4 * wo * wo + ho * ho))
                rows.append({'wave': wave, 'mode': mode, 'pass': leg, 'small_side': wo, 'route': route,
                             'planes': x.shape[0] * P, 'ms': res[k][0], 'range_ms': res[k][1:], 'alg_bytes': nb,
                             'hbm_fraction': nb / (res[k][0] * 1e-3) / HBM_BYTES_PER_S})
                print(json.dumps(rows[-1]))
            del x, c, ll, hi
            torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    dev = 'cuda:0'
    info = gpu_info()
    torch.manual_seed(0)
    x = torch.randn(SHAPE, device=dev)
    N, C, H, W = SHAPE
    rows = []
    for J, wave, mode in CONFIGS:
        f = pw.WPT2DForward(J=J, wave=wave, mode=mode).to(dev)
        i = pw.WPT2DInverse(wave=wave, mode=mode).to(dev)
        fwd1 = pw.DWTForward(J=1, wave=wave, mode=mode).to(dev)
        inv1 = pw.DWTInverse(wave=wave, mode=mode).to(dev)
        L = len(wavelets.Wavelet(wave).dec_lo)
        sizes = packet2d.packet_sizes(H, W, J, L, L, pw.dwt.lowlevel.mode_to_int(mode))
        with torch.no_grad():
            y = f(x)
            assert torch.equal(y, composed_forward(x, fwd1, J)), 'analysis routes differ'
            xr = i(y, size=(H, W))
            xc = composed_inverse(y, inv1, sizes)
            assert (xr - xc).abs().max().item() <= 1e-5 * x.abs().max().item(), 'synthesis routes differ'
            del xr, xc
            # algorithmic bytes: each level's input read once, its output written once
            lv = [4 * N * C * 4 ** j * (sizes[j][0] * sizes[j][1] + 4 * sizes[j + 1][0] * sizes[j + 1][1])
                  for j in range(J)]
            routes = predicted_routes(H, W, J, L, mode, torch.float32)
            for leg, fa, fb in (('forward', lambda: f(x), lambda: composed_forward(x, fwd1, J)),
                                ('inverse', lambda: i(y, size=(H, W)), lambda: composed_inverse(y, inv1, sizes))):
                ma, mb, sa, sb = time_pair(fa, fb, a.iters, a.warmup)
                with _ffi.CallRecorder() as rec:
                    for _ in range(3):
                        fa()
                    per = rec.summary()
                levels = []
                for j in range(J):
                    (h, w), (ho, wo) = sizes[j], sizes[j + 1]
                    tag = ('wpt_afb2d %dx%d L%d' % (h, w, L)) if leg == 'forward' else ('wpt_sfb2d %dx%d L%d' % (ho, wo, L))
                    d = per[tag]
                    route = routes[j] if leg == 'forward' else routes[2 * J - 1 - j]
                    levels.append({'level': j + 1, 'in': [h, w] if leg == 'forward' else [ho, wo],
                                   'out': [ho, wo] if leg == 'forward' else [h, w], 'route': route,
                                   'ms': d['avg_ms'], 'alg_bytes': lv[j],
                                   'hbm_fraction': lv[j] / (d['avg_ms'] * 1e-3) / HBM_BYTES_PER_S})
                nb = sum(lv)
                rows.append({'J': J, 'wave': wave, 'mode': mode, 'pass': leg, 'wpt_ms': ma, 'composed_ms': mb,
                             'wpt_range_ms': sa, 'composed_range_ms': sb, 'speedup': mb / ma, 'alg_bytes': nb,
                             'hbm_fraction': nb / (ma * 1e-3) / HBM_BYTES_PER_S, 'levels': levels})
                print(json.dumps(rows[-1]))
        del y
        torch.cuda.empty_cache()
    del x
    torch.cuda.empty_cache()
    probe = route_probe(dev, a.iters, a.warmup)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'bench_wpt2d.json'), 'w') as fh:
        json.dump({'gpu': info, 'shape': list(SHAPE), 'iters': a.iters, 'rows': rows, 'route_probe': probe}, fh,
                  indent=1)
    print(json.dumps({'gpu': info}))


if __name__ == '__main__':
    main()
