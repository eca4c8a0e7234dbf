"""Generate the second-order gradient golden vectors from the UNMODIFIED reference.

Run in the build container only (needs /root/reference; imports it through oracle/refshim.py with the pywt
stand-in):

    python tests/golden/make_golden_grad2.py

Each ``grad2_*.npz`` (a prefix of its own: other tests collect ``dwt_*``) holds, for one module in float64, the seeded
inputs ``in<i>``, output cotangents ``u<i>`` and input-shaped weights ``w<i>``, and what the reference's autograd
computes from them:

    gx<i>  = grad(f(x), x, u, create_graph=True)
    ggu<i> = grad(gx, u, w)                              (the gradient through the backward pass, w.r.t. u)
    x2_<i> = grad((grad(sum f(x)^2, x, create_graph=True)^2).sum(), x)     (the full second-order chain)

``kind`` is dwt2 (DWTForward, J = 2), idwt2 (DWTInverse of a J = 2 decomposition), dwt1 or idwt1 (the 1-D pair).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import refshim  # noqa: E402

ref = refshim.load()


def module_fn(kind, wave, mode):
    """(f, inputs maker): f maps a list of input tensors to a list of output tensors."""
    if kind == 'dwt2':
        m = ref.DWTForward(J=2, wave=wave, mode=mode)
        return lambda xs: (lambda r: [r[0]] + list(r[1]))(m(xs[0]))
    if kind == 'idwt2':
        m = ref.DWTInverse(wave=wave, mode=mode)
        return lambda xs: [m((xs[0], list(xs[1:])))]
    if kind == 'dwt1':
        m = ref.DWT1DForward(J=2, wave=wave, mode=mode)
        return lambda xs: (lambda r: [r[0]] + list(r[1]))(m(xs[0]))
    m = ref.DWT1DInverse(wave=wave, mode=mode)
    return lambda xs: [m((xs[0], list(xs[1:])))]


def inputs(kind, wave, mode, shape, gen):
    x = torch.randn(*shape, generator=gen, dtype=torch.float64)
    if kind in ('dwt2', 'dwt1'):
        return [x]
    fwd = ref.DWTForward(J=2, wave=wave, mode=mode) if kind == 'idwt2' else ref.DWT1DForward(J=2, wave=wave, mode=mode)
    yl, yh = fwd(x)
    return [torch.randn(t.shape, generator=gen, dtype=torch.float64) for t in [yl] + list(yh)]


def case(kind, wave, mode, shape, seed):
    torch.set_default_dtype(torch.float64)   # the reference's filter buffers follow the default dtype
    gen = torch.Generator().manual_seed(seed)
    f = module_fn(kind, wave, mode)
    xs = [t.requires_grad_(True) for t in inputs(kind, wave, mode, shape, gen)]
    ys = f(xs)
    us = [torch.randn(y.shape, generator=gen, dtype=torch.float64).requires_grad_(True) for y in ys]
    ws = [torch.randn(x.shape, generator=gen, dtype=torch.float64) for x in xs]
    gx = torch.autograd.grad(ys, xs, us, create_graph=True)
    ggu = torch.autograd.grad(gx, us, ws)
    s = sum((y ** 2).sum() for y in f(xs))
    g = torch.autograd.grad(s, xs, create_graph=True)
    x2 = torch.autograd.grad(sum((t ** 2).sum() for t in g), xs)
    d = dict(kind=kind, wave=wave, mode=mode, n_in=len(xs), n_out=len(ys))
    for name, ts in (('in', xs), ('u', us), ('w', ws), ('gx', gx), ('ggu', ggu), ('x2_', x2)):
        for i, t in enumerate(ts):
            d['%s%d' % (name, i)] = t.detach().numpy()
    name = 'grad2_%s_%s_%s' % (kind, wave, mode)
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **{k: np.asarray(v) for k, v in d.items()})
    print(name, [t.shape for t in xs])
    torch.set_default_dtype(torch.float32)


if __name__ == '__main__':
    waves = {'zero': 'db3', 'symmetric': 'db4', 'reflect': 'db3', 'periodic': 'db4', 'periodization': 'db3'}
    k = 0
    for mode, wave in waves.items():
        for kind, shape in (('dwt2', (1, 2, 13, 11)), ('idwt2', (1, 2, 13, 11)), ('dwt1', (2, 2, 21)),
                            ('idwt1', (2, 2, 21))):
            case(kind, wave, mode, shape, 100 + k)
            k += 1
    for kind, shape in (('dwt2', (1, 1, 9, 7)), ('idwt1', (1, 2, 15))):
        case(kind, 'db1', 'symmetric', shape, 100 + k)
        k += 1
