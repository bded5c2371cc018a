"""The RLE1 emit kernel folds each block's CRC into its copy pass: one CTA covers a span of up to four tiles of one
block, and the CRCs of the spans are combined per block.  These cases put block edges where that combination has
seams, and check every block's (raw_start, raw_len, n, crc) and the whole stream against the oracle:
- a block that ends (and so the next one starts) on a span edge, one byte before or after it, and on the first,
  an interior and the last tile edge of a span, at pointer skews 0 and 1;
- a block whose raw span is as long as RLE1 allows at level 9 (one byte value throughout: 51 raw bytes per output
  byte), the length the CRC shift table is sized for;
- a last block shorter than one tile, and an input that ends in a short tile."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import rle1_cases as RC

pytestmark = pytest.mark.gpu
TILE = 4096
SPAN = 4 * TILE


def _run_for_gap(g):
    """Length of a run whose raw bytes exceed its RLE1 output by g (g >= -1)."""
    q = (g + 1) // 250
    return 255 * q + g - 250 * q + 5


def _span_edge_case(target, tail):
    """Level 1: a run, then bytes without runs, so that block 0 ends at span offset `target` (mod SPAN); the last
    block is `tail` bytes long."""
    bs = RC.block_size(1)
    g = (target - bs) % SPAN
    ln = _run_for_gap(g)
    assert ln - RC.outfresh(ln) == g
    body = bytearray(RC._ascii_no_runs(bs + g + 2 * bs + tail, 3 + target))
    RC._plant(body, 0, ln, body[ln + 1] ^ 0x20)
    return bytes(body)


SPAN_TARGETS = [0, 1, SPAN - 1, TILE - 1, TILE, TILE + 1, 2 * TILE, 3 * TILE - 1, 3 * TILE, 3 * TILE + 1, 777]


def _compress_dev(data, level, skew):
    import torch
    from compressjs_b200 import _native
    L = _native.lib()
    buf = torch.zeros(len(data) + 512, dtype=torch.uint8, device="cuda")
    buf[skew:skew + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = L.b2_bzip2_bound(len(data))
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    n = C.c_size_t()
    torch.cuda.synchronize()
    assert L.b2_bzip2_compress_dev(buf.data_ptr() + skew, len(data), level, d_out.data_ptr(), cap, C.byref(n)) == 0, _native.last_error()
    return bytes(d_out[:n.value].cpu().numpy().tobytes())


def _check(data, level, skews=(0,)):
    from compressjs_b200 import _native
    starts, lens, crcs, _ = O.rle1_split(data, level)
    want = [(int(s), int(e) - int(s), int(n), int(c)) for s, e, n, c in zip(starts, list(starts[1:]) + [len(data)], lens, crcs)]
    stream = O.bzip2_compress(data, level)
    for skew in skews:
        z = _compress_dev(data, level, skew)
        got = [(t.raw_start, t.raw_len, t.n, t.crc) for t in _native.last_trace()]
        assert got == want, "skew %d: first differing block %r" % (skew, next(
            (k, a, b) for k, (a, b) in enumerate(zip(got + [None] * len(want), want)) if a != b))
        assert z == stream, "skew %d: stream differs from the oracle's" % skew
    return want


@pytest.mark.parametrize("target", SPAN_TARGETS)
def test_block_edge_in_span(target):
    data = _span_edge_case(target, 100 + target % 7)
    blocks = _check(data, 1, skews=(0, 1))
    assert blocks[1][0] % SPAN == target % SPAN
    assert blocks[-1][1] < TILE and len(data) % TILE


def test_block_at_shift_table_bound():
    bs = RC.block_size(9)
    data = b"a" * (51 * bs + 300) + b"\n" + bytes(RC._ascii_no_runs(5000, 9))
    blocks = _check(data, 9)
    # the first block takes its whole output from the run: 255 raw bytes for every 5 output bytes
    assert blocks[0][1] == RC.cneed(bs) and blocks[0][1] // TILE >= 11200
