"""Time the 3-D DWT's fused kernels against the two-step route (2-D level plus a pass along D) on one GPU.

    python tools/bench_dwt3d.py --out DIR [--iters 20] [--warmup 3]

Workloads: DWT3DForward J = 1 and J = 3 and the matching DWT3DInverse, haar and db4, symmetric mode, float32, on one
large volume pair (2, 1, 512, 512, 512) and on many small volumes (256, 4, 32, 64, 64) -- the two ends of the D-chunk
decision (few volumes march in many D chunks, many volumes in one).  The two routes alternate call by call in the same
run (CUDA events around each call, after warm-up); the report gives the median and spread, the algorithmic bytes (input
read once plus every returned output written once) and their fraction of the 3.35 TB/s data-sheet HBM3 bandwidth, and
the card name, power limit and SM clock read in the same run.  At the timed sizes the routes' analysis outputs must be
equal and their synthesis outputs within twice the per-volume error bound of the tests (tests/oracle3d.py).
Writes DIR/bench_dwt3d.json.
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

HBM_BYTES_PER_S = 3.35e12
SHAPES = {'large': (2, 1, 512, 512, 512), 'small': (256, 4, 32, 64, 64)}


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(','), [v.strip() for v in out.split(',')]))
    except Exception as e:   # (report what failed; the timings stand on their own)
        return {'error': repr(e), 'name': torch.cuda.get_device_name()}


def timed(fn, generic):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if generic:
        with _ffi.generic_kernels():
            e0.record()
            out = fn()
            e1.record()
    else:
        e0.record()
        out = fn()
        e1.record()
    return out, (e0, e1)


def nbytes(*ts):
    return sum(t.numel() * t.element_size() for t in ts if t is not None)


def stats(ms):
    ms = sorted(ms)
    return {'median_ms': ms[len(ms) // 2], 'min_ms': ms[0], 'max_ms': ms[-1], 'n': len(ms)}


def synthesis_bound_ok(y, ref, yl, yh, g0, g1):
    """|y - ref| <= 2 * K * u * G * s per volume (s: max |coefficient| of the volume over every level)."""
    sys.path.insert(0, ROOT)
    from tests import oracle3d
    G, K = oracle3d.bound_sfb3d(g0, g1, True)
    N, C = y.shape[:2]
    s = yl.abs().reshape(N, C, -1).amax(-1)
    for h in yh:
        s = torch.maximum(s, h.abs().reshape(N, C, -1).amax(-1))
    err = (y - ref).abs().reshape(N, C, -1).amax(-1)
    ratio = (err / (2 * K * 2.0 ** -24 * G * s.double().clamp_min(1e-300))).max().item()
    return ratio <= 1.0, ratio


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--shapes', default='large,small')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_dwt3d needs a CUDA device'
    os.makedirs(a.out, exist_ok=True)
    dev = 'cuda'
    res = {'gpu_before': gpu_info(), 'hbm_peak_bytes_per_s': HBM_BYTES_PER_S, 'iters': a.iters, 'runs': []}
    for sname in a.shapes.split(','):
        shape = SHAPES[sname]
        torch.manual_seed(0)
        x = torch.randn(shape, device=dev)
        for wave in ('haar', 'db4'):
            for J in (1, 3):
                f = pw.DWT3DForward(J=J, wave=wave, mode='symmetric').to(dev)
                inv = pw.DWT3DInverse(wave=wave, mode='symmetric').to(dev)
                g0, g1 = inv.g0.cpu().numpy().ravel(), inv.g1.cpu().numpy().ravel()
                with torch.no_grad():
                    for _ in range(a.warmup):
                        for generic in (False, True):
                            timed(lambda: f(x), generic)
                    fw = {False: [], True: []}
                    for _ in range(a.iters):
                        for generic in (False, True):
                            out, ev = timed(lambda: f(x), generic)
                            fw[generic].append(ev)
                    (yl, yh), _ = timed(lambda: f(x), False)
                    (gyl, gyh), _ = timed(lambda: f(x), True)
                    fwd_equal = bool(torch.equal(yl, gyl) and all(torch.equal(p, q) for p, q in zip(yh, gyh)))
                    del gyl, gyh, out
                    for _ in range(a.warmup):
                        for generic in (False, True):
                            timed(lambda: inv((yl, yh)), generic)
                    iv = {False: [], True: []}
                    for _ in range(a.iters):
                        for generic in (False, True):
                            y, ev = timed(lambda: inv((yl, yh)), generic)
                            iv[generic].append(ev)
                    del y
                    y, _ = timed(lambda: inv((yl, yh)), False)
                    gy, _ = timed(lambda: inv((yl, yh)), True)
                    inv_ok, inv_ratio = synthesis_bound_ok(y, gy, yl, yh, g0, g1)
                    torch.cuda.synchronize()
                fbytes = nbytes(x, yl, *yh)
                ibytes = nbytes(yl, *yh, y)
                for kind, evs, b in (('forward', fw, fbytes), ('inverse', iv, ibytes)):
                    for generic in (False, True):
                        st = stats([e0.elapsed_time(e1) for e0, e1 in evs[generic]])
                        st.update({'shape': list(shape), 'wave': wave, 'J': J, 'kind': kind,
                                   'route': 'two_step' if generic else 'fused', 'alg_bytes': b,
                                   'alg_bytes_per_s': b / (st['median_ms'] * 1e-3)})
                        st['fraction_of_hbm_peak'] = st['alg_bytes_per_s'] / HBM_BYTES_PER_S
                        res['runs'].append(st)
                res['runs'][-4]['routes_equal'] = fwd_equal
                res['runs'][-2]['within_bound'] = inv_ok
                res['runs'][-2]['diff_over_bound'] = inv_ratio
                r = res['runs'][-4:]
                print('%-5s %-4s J%d fwd fused %.3f ms (%.0f%% HBM) two-step %.3f ms equal=%s | inv fused %.3f ms '
                      'two-step %.3f ms bound=%s (%.2f)' % (
                          sname, wave, J, r[0]['median_ms'], 100 * r[0]['fraction_of_hbm_peak'], r[1]['median_ms'],
                          fwd_equal, r[2]['median_ms'], r[3]['median_ms'], inv_ok, inv_ratio), flush=True)
                del yl, yh, y, gy
                torch.cuda.empty_cache()
        del x
        torch.cuda.empty_cache()
    res['gpu_after'] = gpu_info()
    with open(os.path.join(a.out, 'bench_dwt3d.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
    ok = all(r.get('routes_equal', True) and r.get('within_bound', True) for r in res['runs'])
    print('outputs check:', 'ok' if ok else 'FAILED')
    return 0 if ok else 1


if __name__ == '__main__':
    sys.exit(main())
