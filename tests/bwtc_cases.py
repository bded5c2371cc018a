"""Case corpus for the BWTC container's models and range coder (csrc/bwtc.cu), built from the model's point of view.

The model sees a block as the symbols of its sentinel BWT column: MTF ranks over the sorted used bytes, zero runs as
RUNA / RUNB digits, rank r as symbol r + 1.  So a case designs a rank sequence and finds an input whose column it is:

1. the ranks run through the inverse MTF (mtfhuff_cases.unmtf) give a column U of n bytes;
2. with the sentinel at row s (the start index the encoder writes), U is the sentinel BWT of some block only when the
   LF permutation over the n + 1 rows is one cycle: mtfhuff_cases.merge_cycles swaps adjacent, different bytes of
   different cycles until it is (the sentinel stays at its row);
3. the block is the inverse sentinel BWT of (U, s), checked by the forward transform.

Blocks are fixed cuts of the raw input, so a multi-block case is its blocks one behind the other, every block but the
last level * 100 000 bytes.  The merge moves a few bytes, and the coder's state carries from block to block, so every
case states what it reaches as predicates over the oracle's trace (oracle.bwtc_compress(trace=True)) and over the
symbols of its blocks; tests/test_bwtc_cases.py asserts them.  Events of the coder that hang on its state (bytes
pending at a block's end, carries at the header or at the finish) are reached by a short tail of random bytes whose seed
was searched for once with `search_seed` and is written down beside the case.
"""
import functools
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle as O
from tests import mtfhuff_cases as MC
from tests import util as U

GROUP = 50            # the zero-run coder's mask words (k_bwtc_widen): bit p % 50 of word p / 50
WIDEN = 16            # symbols per thread of k_bwtc_widen
WARP = 32             # symbols per warp load of k_bwtc_model_fenwick, triples per staged batch of k_bwtc_code
BATCHES = (1, 2, 3)   # B2_BWT_BATCH values whose seams the pending-byte cases sit on


def block_size(level):
    return level * 100000


def old_bound(n):
    """The window size of the parent commit (bwtc_bound): n + n / 8 + (n / 100000 + 2) * 1024 + 64."""
    return n + n // 8 + (n // 100000 + 2) * 1024 + 64


def window_bound(n, nb, level):
    """bwtc_window_bound of csrc/bwtc.cu: the most coded bytes of nb blocks of n raw bytes."""
    return (2 if level <= 5 else 3) * n + n // 64 + nb * 1024 + 64


# ---- blocks from ranks ---------------------------------------------------------------------------------------------
def symbols(U_):
    """The model's symbols of a sentinel BWT column (lib/BWTC.js:93-137): MTF over the sorted used bytes, zero runs
    as bijective base-2 digits (0 = RUNA, 1 = RUNB), rank r as r + 1."""
    ranks = MC.mtf_ranks(U_) if len(U_) else np.zeros(0, np.int32)
    out, run = [], 0
    for r in ranks.tolist() + [-1]:
        if r == 0:
            run += 1
            continue
        while run:
            if run & 1:
                out.append(0)
                run -= 1
            else:
                out.append(1)
                run -= 2
            run >>= 1
        if r > 0:
            out.append(r + 1)
    return np.array(out, np.int32)


def block_from_ranks(ranks, used, sentinel=None):
    """Raw block whose sentinel BWT column has MTF ranks `ranks` over `used` (up to the swaps of the cycle merge), with
    the sentinel at row `sentinel` (default n / 3)."""
    n = len(ranks)
    s = n // 3 + 1 if sentinel is None else sentinel
    Ucol, _ = MC.merge_cycles(MC.unmtf(np.asarray(ranks, np.int32), used), sentinel=s)
    T = O.unbwt_sentinel(Ucol.tobytes(), s)
    assert O.bwt_sentinel(T) == (Ucol.tobytes(), s)
    return T


def cycling_ranks(n):
    """Ranks 1, 2, ..., 255, 1, 2, ...: over 256 bytes every symbol comes back just after its weight was halved."""
    return 1 + np.arange(n) % 255


def random_ranks(n, alpha, seed, p=0.3):
    """Every byte of the alphabet brought to the front once, then geometric ranks with zero runs."""
    g = U.rng(seed)
    r = np.minimum(g.geometric(p, size=n), alpha) - 1
    head = np.full(alpha, alpha - 1)   # rank alpha - 1 brings the least recent byte to the front: all of them in turn
    return np.concatenate([head, r[:max(n - head.size, 0)]]).astype(np.int32)


def first_coder_byte(n):
    """Index of the coder's first byte in the stream of n raw bytes: behind "bwtc" and the written size groups."""
    return 4 + (max(n + 1, 1).bit_length() + 6) // 7 - 1


def tail(seed, k):
    return U.rng(seed).integers(0, 256, size=k, dtype=np.uint8).tobytes()


@functools.lru_cache(maxsize=None)
def worst_block(level):
    return block_from_ranks(cycling_ranks(block_size(level)), list(range(256)))


# ---- cases ---------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    build: object          # () -> raw input
    levels: tuple
    claims: list = field(default_factory=list)   # (what, predicate(info, level))


class CaseInfo:
    """The oracle's stream and trace of one case at one level, and the symbols of its blocks."""

    def __init__(self, raw, level):
        self.raw, self.level = raw, level
        self.z, self.blocks, self.file = O.bwtc_compress(raw, level, trace=True)

    @functools.cached_property
    def syms(self):
        bs = block_size(self.level)
        return [symbols(np.frombuffer(O.bwt_sentinel(self.raw[k:k + bs])[0], np.uint8)) for k in range(0, len(self.raw), bs)]

    def coded(self):
        """Coded bytes of the blocks: the stream without the header's written size groups and the trailer."""
        return len(self.z) - (len(O.bwtc_compress(b"", self.level)) - 5) - 5


def every(f):
    return lambda ci: any(f(b) for b in ci.blocks)


def seam(B, f):
    """f holds at the end of a block that ends a batch of B blocks and is not the last block."""
    return lambda ci: any(f(b) for k, b in enumerate(ci.blocks[:-1]) if (k + 1) % B == 0)


def sym256_at(pred):
    return lambda ci: any(pred(np.flatnonzero(s == 256)).any() for s in ci.syms)


def _alphabet(alpha, n, seed):
    if alpha == 1:
        return b"q" * n
    return block_from_ranks(random_ranks(n, alpha, seed), MC.used_bytes(alpha, seed))


def _tuned(make, pick, lo, hi):
    """make(n) for the first n in [lo, hi) whose level-9 trace satisfies pick(block 0)."""
    for n in range(lo, hi):
        raw = make(n)
        if pick(O.bwtc_compress(raw, 9, trace=True)[1][0]):
            return raw
    raise AssertionError("no length in [%d, %d) reaches the target" % (lo, hi))


def search_seed(make, ok, level, seeds=range(4096)):
    """The first seed whose input make(seed) satisfies ok(CaseInfo): how the seeds written beside the cases were found."""
    for s in seeds:
        ci = CaseInfo(make(s), level)
        if ok(ci):
            return s
    raise AssertionError("no seed reaches the target")


def _seams_input(seeds, level=1):
    """Full blocks of random bytes whose last 16 raw bytes come from seeds[k], then a short
    last block: the bytes pending at each block's end hang on its tail."""
    bs = block_size(level)
    base = tail(500, bs)
    blocks = [base[:-16] + tail(s, 16) for s in seeds]
    return b"".join(blocks) + _alphabet(64, 5000, 501)


# Found with search_seed, block by block (each block's seed with the ones before it fixed): in SEAMS_PLAIN, bytes pending
# at the end of blocks 0, 1 and 2 (seams of batches of 1, 2 and 3 blocks), each resolved in the next block without a
# carry (as FF bytes); in SEAMS_CARRY, bytes pending at the end of block 0 resolved in block 1 by a carry (as 00 bytes),
# about one seed in 2000.
SEAMS_CARRY = (270, 0, 0)
SEAMS_PLAIN = (180, 401, 38)
# Sizes with size + 1 = 127 (mod 128): the size field ends in the group 0x7F, 0xFF with its flag, which the coder holds
# as its first `buffer`.  No carry can reach it: the level byte is coded first (tot 256, from low = 0, range = 2^31), so
# low = level * 2^23 and range = 2^23 when the next triple normalises, and the buffer goes out as it is.  The cases check
# that the 0xFF goes out unchanged (and 0x80 in the stream without a size).
HEADER_SIZES = ((126, 1), (126, 9), (100094, 1), (100094, 9))
# The trailer: a carry at the finish; the rounding rule taken and not taken.
FINISH = {"carry": 20, "round": 0, "noround": 56}


@functools.lru_cache(maxsize=1)
def cases():
    cs = []
    for a in (1, 2, 3, 31, 32, 33, 63, 64, 127, 128, 129, 255, 256):
        cs.append(Case("alphabet_%d" % a, (lambda a=a: _alphabet(a, 6000, a)), (1, 9),
                       [("alphabet %d" % a, lambda ci, a=a: ci.blocks[0].alpha == a)]))
    for r in (0, 1, 31):
        cs.append(Case("nsym_%d_mod32" % r,
                       (lambda r=r: _tuned(lambda n: _alphabet(40, n, 900), lambda b: b.nsym % WARP == r, 3000, 3100)),
                       (9,), [("symbols = %d (mod 32)" % r, lambda ci, r=r: ci.blocks[0].nsym % WARP == r)]))
    for r in (0, 1, 31):
        cs.append(Case("triples_%d_mod32" % r,
                       (lambda r=r: _tuned(lambda n: _alphabet(40, n, 901), lambda b: b.ntriples % WARP == r, 3000, 3100)),
                       (9,), [("triples = %d (mod 32)" % r, lambda ci, r=r: ci.blocks[0].ntriples % WARP == r)]))
    fen = [("a rescale at exactly 0xFF00", every(lambda b: b.rescales_ff00 > 0)),
           ("a rescale triggered by an escape step, the literal coded after it", every(lambda b: b.rescales_esc > 0)),
           ("an escape as the 32nd symbol of a warp load", every(lambda b: b.esc_lane31 > 0)),
           ("a re-escape (a seen symbol halved back to unseen: 9 rescales without it)", every(lambda b: b.reescapes > 0)),
           ("1 correction step of the reciprocal", every(lambda b: b.corr[1] > 0)),
           ("0 correction steps of the reciprocal", every(lambda b: b.corr[0] > 0)),
           ("a pending run of 2 bytes", lambda ci: ci.file.max_help >= 2)]
    cs.append(Case("random_l9", lambda: U.rng(77).integers(0, 256, 600000, dtype=np.uint8).tobytes(), (6, 9), fen))
    cs.append(Case("last_escape_then_noescape", lambda: _alphabet(6, 200000, 6), (9,),
                   [("the last escape", every(lambda b: b.last_escape > 0)),
                    ("a rescale with noEscape after it", every(lambda b: b.rescales_noesc > 0))]))
    cs.append(Case("deferred_sum", lambda: U.rng(78).integers(0, 256, 250000, dtype=np.uint8).tobytes(), (1, 5),
                   [("a table rebuild", every(lambda b: b.ds_rebuilds > 0)),
                    ("update[esc] capped at 40", every(lambda b: b.ds_esc_cap > 0)),
                    ("escapes and re-escapes", every(lambda b: b.escapes > 0 and b.reescapes > 0)),
                    ("1 correction step of the reciprocal", every(lambda b: b.corr[1] > 0))]))
    s256 = [("symbol 256 at p = 0 (mod 16)", sym256_at(lambda p: p % WIDEN == 0)),
            ("symbol 256 at p = 15 (mod 16)", sym256_at(lambda p: p % WIDEN == WIDEN - 1)),
            ("symbol 256 at the first symbol of a mask group", sym256_at(lambda p: p % GROUP == 0)),
            ("symbol 256 at the last symbol of a mask group", sym256_at(lambda p: p % GROUP == GROUP - 1)),
            ("symbol 256 at bit 50..63 of a 64-bit word's position (p % 64 >= 50)", sym256_at(lambda p: p % 64 >= GROUP))]

    def slots():
        """Blocks with symbol 256, without it, and with it elsewhere: every slot of batches of 1, 2 and 3 blocks sees a
        block with symbol 256 after one with it at other positions, and after one without it."""
        a = block_from_ranks(random_ranks(block_size(1), 256, 31, p=0.02), list(range(256)))
        b = block_from_ranks(random_ranks(block_size(1), 256, 32, p=0.02), list(range(256)))
        c = _alphabet(200, block_size(1), 33)
        return a + b + c + a + b + c + b + a + b[:40000]
    def slot_claim(B):
        def f(ci):
            has = [bool((s == 256).any()) for s in ci.syms]
            pos = [frozenset(np.flatnonzero(s == 256).tolist()) for s in ci.syms]
            after_other = any(has[k] and has[k - B] and pos[k] - pos[k - B] for k in range(B, len(has)))
            after_none = any(has[k] and not has[k - B] for k in range(B, len(has)))
            return after_other and after_none
        return ("batches of %d: a slot's block with symbol 256 after one with it elsewhere, and after one without it" % B, f)
    cs.append(Case("symbol_256_slots", slots, (1,), s256 + [slot_claim(B) for B in BATCHES]))
    cs.append(Case("pending_at_seams_carry", lambda: _seams_input(SEAMS_CARRY), (1,),
                   [("bytes pending at the end of block 0, resolved in block 1 by a carry",
                     lambda ci: ci.blocks[0].help >= 1 and ci.blocks[1].resolved_in == 2)]))
    cs.append(Case("pending_at_seams_plain", lambda: _seams_input(SEAMS_PLAIN), (1,),
                   [("bytes pending at the seam of batches of %d" % B, seam(B, lambda b: b.help >= 1)) for B in BATCHES] +
                   [("the bytes pending at the end of blocks 0, 1 and 2 resolved without a carry",
                     lambda ci: all(ci.blocks[k + 1].resolved_in == 1 for k in range(3)))]))
    for n, lv in HEADER_SIZES:
        cs.append(Case("header_ff_%d_l%d" % (n, lv), (lambda n=n: tail(n, n)), (lv,),
                       [("size + 1 = 127 (mod 128)", lambda ci, n=n: (n + 1) % 128 == 127),
                        ("the coder's first byte is the size field's last group, 0xFF", lambda ci: ci.z[first_coder_byte(len(ci.raw))] == 0xFF),
                        ("no carry into it", lambda ci: ci.file.first_carry == 0)]))
    cs.append(Case("finish_carry", lambda: tail(FINISH["carry"], 3000), (9,),
                   [("a carry at the finish", lambda ci: ci.file.finish_carry == 1)]))
    cs.append(Case("finish_round", lambda: tail(FINISH["round"], 3000), (9,),
                   [("the rounding rule adds one", lambda ci: ci.file.finish_round == 1)]))
    cs.append(Case("finish_noround", lambda: tail(FINISH["noround"], 3000), (9,),
                   [("the rounding rule adds nothing", lambda ci: ci.file.finish_round == 0)]))
    cs.append(Case("bytecount_wraps", lambda: U.rng(79).integers(0, 256, 17 << 20, dtype=np.uint8).tobytes(), (1,),
                   [("more than 2^24 coded bytes", lambda ci: ci.file.bytecount > 1 << 24)]))
    grow = [("grows past the parent's window bound", lambda ci: ci.coded() > old_bound(len(ci.raw)))]
    for lv in (6, 9):
        cs.append(Case("worst_growth_l%d" % lv, (lambda lv=lv: worst_block(lv)), (lv,), grow))
        cs.append(Case("worst_growth_l%d_x3" % lv, (lambda lv=lv: worst_block(lv) * 3), (lv,), grow))
    # The deferred-sum model codes the cycling ranks at 1.001 n: its worst growth found is that of random bytes.
    cs.append(Case("worst_growth_l5", lambda: U.rng(80).integers(0, 256, 500000, dtype=np.uint8).tobytes(), (5,),
                   [("grows by 2 %", lambda ci: ci.coded() > 1.02 * len(ci.raw))]))
    return cs


def case(name):
    return next(c for c in cases() if c.name == name)


@functools.lru_cache(maxsize=None)
def raw(name):
    return bytes(case(name).build())


@functools.lru_cache(maxsize=None)
def info(name, level):
    return CaseInfo(raw(name), level)
