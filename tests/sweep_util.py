"""Helpers shared by the streaming-kernel boundary sweeps (tests/test_gpu_dtcwt_stream_sweep.py,
tests/test_gpu_dwt_stream_sweep.py): the row-chunk rule of the launchers, canaried NaN-filled output buffers, and kernel
names read from a torch.profiler trace.  Importable without a GPU."""
import re

import numpy as np
import torch


def pick_chunks(base_items, rows_out, min_rows, pro, conc):
    """stream_common.cuh pick_chunks: the number of row chunks of each (plane, strip) march."""
    max_chunks = (rows_out + min_rows - 1) // min_rows
    best, best_nc, last_ch = 0.0, 1, -1
    for nc in range(1, min(max_chunks, 64) + 1):
        ch = -(-rows_out // nc)
        ch = -(-ch // min_rows) * min_rows
        if ch == last_ch:
            continue
        last_ch = ch
        n = -(-rows_out // ch)
        cost = base_items * (rows_out + n * pro) / max(conc, 1) + 0.5 * (ch + pro)
        if nc == 1 or cost < best:
            best, best_nc = cost, n
    return best_nc


# resident one-warp CTAs on an H100: 1 .. 32 per SM on 132 SMs, whatever the kernel's occupancy
CONC_RANGE = range(132, 132 * 32 + 1, 132)


def chunk_range(base_items, rows_out, min_rows, pro):
    """(min, max) chunk count over every occupancy in CONC_RANGE."""
    counts = [pick_chunks(base_items, rows_out, min_rows, pro, c) for c in CONC_RANGE]
    return min(counts), max(counts)


MANY_CHUNKS = 'many chunks'     # 1 x 2 tall planes: every march splits into many row chunks at any occupancy
ONE_CHUNK = 'one chunk'         # 2000 small planes: every march is one chunk


# ---- unwritten outputs and stray writes -------------------------------------------------------------------------------

PAD = 77
CANARY = 7.5


class Canaried(object):
    """A device buffer of `shape` filled with NaN, between PAD canary values on each side."""

    def __init__(self, shape, dev='cuda'):
        n = int(np.prod(shape))
        self.buf = torch.full((n + 2 * PAD,), CANARY, device=dev)
        self.buf[PAD:PAD + n] = float('nan')
        self.t = self.buf[PAD:PAD + n].view(shape)

    def ptr(self):
        return self.t.data_ptr()

    def check_canaries(self, what):
        assert bool((self.buf[:PAD] == CANARY).all()) and bool((self.buf[-PAD:] == CANARY).all()), what + ': canary'

    def check(self, what):
        self.check_canaries(what)
        assert not bool(torch.isnan(self.t).any()), what + ': unwritten outputs'


# ---- kernel names in a profiler trace ---------------------------------------------------------------------------------

def kernel_namer(stream_names, tile_names):
    """A function mapping a demangled CUDA kernel name to '<stream kernel><template args without spaces>',
    '<tile>_tile' (for k_<tile>_tile), or None for any other kernel."""
    rx = re.compile(r'(%s)<([^>]*)>|k_(%s)_tile' % ('|'.join(stream_names), '|'.join(tile_names)))

    def short(name):
        m = rx.search(name)
        if not m:
            return None
        if m.group(1):
            return '%s<%s>' % (m.group(1), m.group(2).replace(' ', ''))
        return m.group(3) + '_tile'
    return short


def traced_kernels(run, short):
    """Call run() under a torch.profiler CUDA trace; the short names (in launch order) of the kernels `short` knows, or
    None when CUDA activity tracing is unavailable or recorded nothing."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        events = [e for e in prof.events() if short(e.name) is not None]
    except Exception:   # (no CUPTI on this machine)
        return None
    if not events:
        return None
    return [short(e.name) for e in sorted(events, key=lambda e: e.time_range.start)]
