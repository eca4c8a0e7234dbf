"""Case matrix of the DWT boundary sweep (tests/test_gpu_dwt_stream_sweep.py) and the dispatch rules that predict which
kernel each case launches.  No GPU needed: tests/test_dwt_sweep_matrix.py checks on the CPU that the matrix reaches every
instantiation and both row-chunk regimes.

Instantiations (72):
  afb2d_stream<L, 32, MINB, 2, XM>   L = 2..20 even; XM 0 (zero / symmetric / reflect), 1 (periodic), 2 (periodization);
                                     MINB = 12 for XM = 0 and L >= 14, else 1                                    (30)
  sfb2d_stream<L, PER>               L = 2..20, PER = periodization                                              (20)
  sfb2d_stream4<L>                   L = 2..8, non-periodization planes with more than 64 output column pairs     (4)
  dwt_pyramid<L, MAXT, MINB, SPLIT>  L = 2..12; MAXT 160 (MINB pyr_minb_small(L), SPLIT pyr_split(L)), 256 (2, 1),
                                     512 (1, 1)                                                                    (18)
dwt_pyramid<10, 512, 1, 1> cannot run on a device with 227 KB of shared memory per block: a 10-tap stage is 10 rows, and
every plan the policy asks for that needs more than six worker warps (one level over 576 columns, or several levels from
512 columns) needs more shared memory than that for its input ring and staging rings.  UNREACHABLE names it; the CPU test checks it against the
shipped plan."""
from oracle import oracle as orc
from tests import sweep_util
from tests.sweep_util import MANY_CHUNKS, ONE_CHUNK

LS = list(range(2, 21, 2))
PYR_LS = [2, 4, 6, 8, 10, 12]
XM_MODES = {0: ('symmetric', 'zero', 'reflect'), 1: ('periodic',), 2: ('periodization',)}
SYN_MODES = ('zero', 'symmetric', 'reflect', 'periodic')     # every non-periodization mode synthesises alike
PYR_MODES = ('symmetric', 'zero', 'reflect')


def _xm(mode):
    return {'periodic': 1, 'periodization': 2}.get(mode, 0)


def afb_name(L, mode):
    xm = _xm(mode)
    return 'afb2d_stream<%d,32,%d,2,%d>' % (L, 12 if (xm == 0 and L >= 14) else 1, xm)


def pyr_hs(L):
    m = 1
    while (L // 2) * m < 4 or ((L // 2) * m) & 1:
        m += 1
    return (L // 2) * m


def pyr_name(L, threads):
    if threads <= 160:
        return 'dwt_pyramid<%d,160,%d,%d>' % (L, 4 if L <= 8 else 3, 2 if pyr_hs(L) % 4 == 0 else 1)
    if threads <= 256:
        return 'dwt_pyramid<%d,256,2,1>' % L
    return 'dwt_pyramid<%d,512,1,1>' % L


ALL_KERNELS = ([afb_name(L, m) for L in LS for m in ('symmetric', 'periodic', 'periodization')] +
               ['sfb2d_stream<%d,%s>' % (L, p) for L in LS for p in ('false', 'true')] +
               ['sfb2d_stream4<%d>' % L for L in (2, 4, 6, 8)] +
               [pyr_name(L, t) for L in PYR_LS for t in (160, 256, 512)])
UNREACHABLE = ['dwt_pyramid<10,512,1,1>']


def _ceil(a, b):
    return -(-a // b) * b


# ---- analysis: one level, afb2d_level --------------------------------------------------------------------------------
# strips of 64 output columns, chunks of 16 output rows.  Output widths: below one strip, one strip, one strip + 1,
# several strips with a partial last one, 64k + 1 (a one-column last strip whose mirror source lies left of its window:
# widen_left).  Input widths alternate between odd and even (2 mod 4 or 0 mod 4), read through a row pitch rounded up to
# 32 floats, as levels >= 2 read the inter-level workspace.  Ho = 37: chunks 16 + 16 + 5.
AFB_WO = [40, 64, 65, 200, 129]
_DEF = dict(pitch=None, rows_pad=0, offset=0, lw=None, has_hi=True, crop=None, ll_trim=False, regime=None,
            canary=False, label=None)


def _case(family, L, mode, shape, **kw):
    c = dict(_DEF, family=family, L=L, mode=mode, shape=tuple(shape))
    c.update(kw)
    c['id'] = '%s-L%d-%s-%s' % (family, L, mode, 'x'.join(map(str, shape)))
    for k in ('J', 'pitch', 'rows_pad', 'offset', 'lw', 'has_hi', 'crop', 'll_trim', 'regime', 'label'):
        if k in c and c[k] != _DEF.get(k, None):
            c['id'] += '-%s=%s' % (k, str(c[k]).replace(' ', ''))
    return c


def _afb_in(n_out, L, mode, odd):
    """An input length with coefficient length n_out: the odd one or the even one."""
    if mode == 'periodization':
        n = 2 * n_out - 1
    else:
        n = 2 * n_out - L + 1
    return n if (n % 2 == 1) == odd else n + 1


def afb_cases():
    out = []
    for L in LS:
        for xm, modes in XM_MODES.items():
            for mi, mode in enumerate(modes):
                for k, wo in enumerate(AFB_WO):
                    W = _afb_in(wo, L, mode, odd=(k + mi) % 2 == 0)
                    H = _afb_in(37, L, mode, odd=(k % 2 == 1))
                    out.append(_case('afb', L, mode, (2, 3, H, W), pitch=_ceil(W, 32), canary=(k == 4 and mi == 0)))
    for L in (8, 16):
        W = _afb_in(130, L, 'symmetric', True)
        out.append(_case('afb', L, 'symmetric', (1, 2, _afb_in(420, L, 'symmetric', True), W), pitch=_ceil(W, 32),
                         regime=MANY_CHUNKS))
        W = _afb_in(40, L, 'zero', True)
        out.append(_case('afb', L, 'zero', (1000, 2, _afb_in(14, L, 'zero', False), W), pitch=_ceil(W, 32),
                         regime=ONE_CHUNK))
    W = _afb_in(129, 6, 'symmetric', True)
    out += [
        # plane stride (H + 3) * pitch: the planes of a taller buffer
        _case('afb', 6, 'symmetric', (1, 6, 75, W), pitch=_ceil(W, 32), rows_pad=3),
        _case('afb', 12, 'reflect', (1, 6, 75, 200), rows_pad=3),
        # fallbacks to the generic kernel: a row pitch that is not a multiple of 4 floats; filters of different lengths
        # along W and H (the row/col naming quirk of the reference makes those reachable)
        _case('afb', 8, 'symmetric', (2, 3, 75, 251), label='fallback'),
        _case('afb', 4, 'zero', (2, 3, 75, 131), pitch=132, lw=6, label='fallback'),
    ]
    return out


# ---- synthesis: one level, sfb2d_level -------------------------------------------------------------------------------
# sfb2d_stream: strips of 64 output column pairs; sfb2d_stream4 (L <= 8, more than 64 pairs): strips of 128 pairs.
# Output column pairs: 20, 64 | 65 (2-column -> wide kernel), 128 | 129 (one wide strip, + a one-pair remainder).
SFB_NP = [20, 64, 65, 128, 129]
PER_WC = [None, 64, 65, 200]       # None: below L / 2 coefficients


def sfb_cases():
    out = []
    for L in LS:
        for k, npairs in enumerate(SFB_NP):
            mode = SYN_MODES[(k + L // 2) % 4]
            Wc = npairs + L // 2 - 1
            out.append(_case('sfb', L, mode, (2, 3, 19 + k % 2, Wc), canary=(npairs == 20 or (L <= 8 and npairs == 129))))
        # AFB2D.backward crops the output to the analysis input: odd crops, and one that moves a plane from 65 to 64
        # output column pairs (wide -> 2-column kernel for L <= 8)
        Wc = 65 + L // 2 - 1
        Ho, Wo = 2 * 20 - L + 2, 2 * Wc - L + 2
        out.append(_case('sfb', L, 'symmetric', (2, 3, 20, Wc), crop=(Ho - 1, Wo - 1)))
        out.append(_case('sfb', L, 'zero', (2, 3, 20, Wc), crop=(Ho - 3, 128)))
        for k, wc in enumerate(PER_WC):
            Wc = wc if wc is not None else max(1, L // 2 - 1)
            out.append(_case('sfb', L, 'periodization', (2, 3, 7 if k == 0 else 19, Wc), canary=(k == 3)))
        out.append(_case('sfb', L, 'periodization', (2, 3, 19, 65), crop=(37, 129)))
    out += [
        _case('sfb', 8, 'symmetric', (2, 3, 19, 132), has_hi=False),
        _case('sfb', 14, 'zero', (2, 3, 19, 90), has_hi=False),
        _case('sfb', 6, 'periodization', (2, 3, 19, 70), has_hi=False),
        # DWTInverse trims the low-pass by one row and one column: a view with row pitch Wc + 1
        _case('sfb', 8, 'symmetric', (2, 3, 19, 132), ll_trim=True),
        _case('sfb', 12, 'reflect', (2, 3, 19, 70), ll_trim=True),
        _case('sfb', 4, 'periodization', (2, 3, 19, 131), ll_trim=True),
        _case('sfb', 4, 'symmetric', (1, 2, 400, 66), regime=MANY_CHUNKS),
        _case('sfb', 12, 'zero', (1, 2, 400, 70), regime=MANY_CHUNKS),
        _case('sfb', 8, 'periodization', (1, 2, 400, 70), regime=MANY_CHUNKS),
        _case('sfb', 4, 'symmetric', (1000, 2, 10, 66), regime=ONE_CHUNK),
        _case('sfb', 12, 'zero', (1000, 2, 10, 30), regime=ONE_CHUNK),
        _case('sfb', 8, 'periodization', (1000, 2, 10, 24), regime=ONE_CHUNK),
        _case('sfb', 4, 'symmetric', (2, 3, 19, 70), lw=6, label='fallback'),   # filters of different lengths
    ]
    return out


# ---- the whole forward transform: dwt_forward_levels (b200w_dwt_forward) -------------------------------------------------

def _levels(H, W, J, L, mode):
    sizes = []
    for _ in range(J):
        H, W = orc.coeff_len(H, L, mode), orc.coeff_len(W, L, mode)
        sizes.append((H, W))
    return sizes


def odd_width(L, J, W0, mode='symmetric'):
    """The smallest W >= W0, W % 4 == 0, whose levels >= 2 (and level 1 where W % 4 == 0 allows it) are all odd."""
    W = _ceil(W0, 4)
    while True:
        ws = [w for _, w in _levels(64, W, J, L, mode)]
        if all(w % 2 == 1 for w in ws[1:]) and (ws[0] % 2 == 1 or (L // 2) % 2 == 1):
            return W
        W += 4


def pyr_cases():
    out = []
    for L in PYR_LS:
        m = PYR_MODES[L // 2 % 3]
        n = PYR_MODES[(L // 2 + 1) % 3]
        out += [
            _case('pyr', L, m, (2, 3, 37, 132), J=1, canary=True),                       # one level, 160 threads
            _case('pyr', L, n, (2, 2, 23, 600), J=1, canary=True),                       # one level, 256 threads
            _case('pyr', L, m, (2, 2, 64, odd_width(L, 4, 512)), J=4, canary=True),      # fused J = 4
            _case('pyr', L, n, (2, 3, 40, odd_width(L, 2, 200)), J=2, canary=True),      # level 1 fused, W < 512
            _case('pyr', L, m, (2, 3, 41, odd_width(L, 3, 300)), J=3),
            _case('pyr', L, n, (2, 2, 30, odd_width(L, 3, 512)), J=3),
            # plan edges: level 2 exactly L rows (accepted), one row short (level 1 only); level 1 exactly L rows
            _case('pyr', L, m, (2, 2, L + 1, 516), J=2),
            _case('pyr', L, m, (2, 2, L, 516), J=2, label='edge'),
            _case('pyr', L, n, (2, 3, L, 132), J=1),
        ]
        if L >= 4:
            out.append(_case('pyr', L, n, (2, 3, L - 1, 132), J=1, label='edge'))    # level 1 one row short
        if L % 4 == 0:
            out.append(_case('pyr', L, m, (2, 3, 20, L), J=1))                         # level 1 exactly L columns
        if L % 4 == 2 and L > 2:
            out.append(_case('pyr', L, m, (2, 3, 20, L - 2), J=1, label='edge'))      # two columns short
    W = odd_width(8, 3, 512)
    out += [
        _case('pyr', 8, 'symmetric', (2, 3, 40, W), J=3, pitch=W + 32),                 # input pitch > W
        _case('pyr', 8, 'symmetric', (1, 3, 40, W), J=3, rows_pad=3),                   # plane stride (H + 3) * W
        _case('pyr', 8, 'symmetric', (1, 3, 40, W), J=3, offset=40 * W),               # a channel slice
        _case('pyr', 8, 'zero', (2, 3, 40, W), J=3, offset=4, canary=True),              # 16- but not 128-byte aligned
        _case('pyr', 8, 'zero', (2, 3, 40, W), J=3, offset=1, canary=True, label='edge'),  # 4-byte aligned: level kernels
        _case('pyr', 4, 'reflect', (2, 3, 40, 260), J=2, pitch=292, canary=True),
        _case('pyr', 4, 'reflect', (2, 3, 40, 260), J=2, offset=4),
        _case('pyr', 4, 'reflect', (2, 3, 40, 260), J=2, offset=2, label='edge'),
    ]
    return out


CASES = afb_cases() + sfb_cases() + pyr_cases()


# ---- dispatch rules ----------------------------------------------------------------------------------------------------

def layout(c):
    """(plane stride, row pitch, base offset in floats) of the case's input (analysis / pyramid)."""
    N, C, H, W = c['shape']
    pitch = c['pitch'] or W
    return (H + c['rows_pad']) * pitch, pitch, c['offset']


def _plan(c, J, ll_pitch=0):
    from tests.emu import emu_backend as eb
    N, C, H, W = c['shape']
    ps, pitch, off = layout(c)
    # emu_plan_pyramid checks a 16-byte aligned pointer and a plane stride of H * pitch: the rest of the alignment rule
    # (plan_pyramid: x % 16, xps % 4) is applied here
    if (off * 4) % 16 or ps % 4:
        return None
    return eb.plan_pyramid(N * C, H, W, J, c['L'], c['mode'], xpitch=pitch, ll_pitch=ll_pitch)


def dwt_policy(c):
    """b200wave.cu dwt_policy: ('all' | 'first' | 'levels', plan)."""
    N, C, H, W = c['shape']
    J = c['J']
    if (J == 1 or W >= 512):
        p = _plan(c, J)
        if p is not None:
            return 'all', p
    if J >= 2:
        wo = orc.coeff_len(W, c['L'], c['mode'])
        p = _plan(c, 1, _ceil(wo, 32))
        if p is not None:
            return 'first', p
    return 'levels', None


def aligned(c):
    ps, pitch, off = layout(c)
    return ps % 4 == 0 and pitch % 4 == 0 and (off * 4) % 16 == 0


def sfb_name(c):
    L, mode, (N, C, Hc, Wc) = c['L'], c['mode'], c['shape']
    if c['lw']:
        return 'sfb2d_tile'
    if mode == 'periodization':
        return 'sfb2d_stream<%d,true>' % L
    Wo = orc.rec_len(Wc, L, mode)
    if c['crop']:
        Wo = min(Wo, c['crop'][1])
    if L <= 8 and (Wo + 1) // 2 > 64:
        return 'sfb2d_stream4<%d>' % L
    return 'sfb2d_stream<%d,false>' % L


def expected_kernels(c):
    """The kernels one call of the case launches, in order."""
    fam, L = c['family'], c['L']
    if fam == 'afb':
        return [afb_name(L, c['mode']) if (aligned(c) and not c['lw']) else 'afb2d_tile']
    if fam == 'sfb':
        return [sfb_name(c)]
    pol, plan = dwt_policy(c)
    rest = [afb_name(L, c['mode'])] * (c['J'] - 1)     # levels >= 2 read the aligned workspace
    if pol == 'all':
        return [pyr_name(L, plan['threads'])]
    if pol == 'first':
        return [pyr_name(L, plan['threads'])] + rest
    return [afb_name(L, c['mode']) if aligned(c) else 'afb2d_tile'] + rest


def chunk_counts(c):
    """(min, max) row chunks of each (plane, strip) march of a streaming analysis / synthesis case, over every occupancy."""
    N, C, H, W = c['shape']
    L, mode = c['L'], c['mode']
    if c['family'] == 'afb':
        Ho, Wo = orc.coeff_len(H, L, mode), orc.coeff_len(W, L, mode)
        return sweep_util.chunk_range(N * C * -(-Wo // 64), Ho, 16, (L - 2) // 2 + 8)
    name = sfb_name(c)
    if mode == 'periodization':
        pairs_w, pairs_h = W, H
    else:
        Ho, Wo = orc.rec_len(H, L, mode), orc.rec_len(W, L, mode)
        if c['crop']:
            Ho, Wo = min(Ho, c['crop'][0]), min(Wo, c['crop'][1])
        pairs_w, pairs_h = (Wo + 1) // 2, (Ho + 1) // 2
    strips = -(-pairs_w // (128 if name.startswith('sfb2d_stream4') else 64))
    return sweep_util.chunk_range(N * C * strips, pairs_h, 16, L // 2 + 8)
