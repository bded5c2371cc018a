"""Inputs that put the libbz2 flavor's block cut and table search on their corners.

Every case is (name, data, level).  ``cut_cases`` plant a piece of a chosen length at the first block's cut; each comes
with the corner it must hit, asserted from the model (``check_cut_case``).  ``table_cases`` are single blocks whose
zero-run coder output sits on an nGroups threshold, whose initial partition takes the odd-nPart step, with alphabets of
1 and 256 bytes, or periodic (equal rotations: the origPtr tie rule) (``check_table_case``).  All are seeded, so the GPU tests and the golden file see the same bytes.
"""
import numpy as np

from tests import libbz2_model as M


def nmax(level):
    return 100000 * level - 19


def run_free(n, seed):
    """n bytes, no two neighbours equal: every byte is a piece of one."""
    r = np.random.default_rng(seed).integers(1, 256, n, dtype=np.int64)
    return (np.cumsum(r) % 256).astype(np.uint8).tobytes()


def _tail(seed):
    return run_free(3000, seed)


def _rle(length):
    return length if length < 4 else 5


def cut_cases():
    """(name, data, level, expect): expect = (first block's RLE1 size, first block's raw length) or None."""
    out = []
    lv = 1
    nm = nmax(lv)
    # the closing piece (5 equal bytes) ends exactly on nblockMAX, and 1..4 bytes past it
    for past in range(5):
        p = nm + past - 5
        head = run_free(p, 10 + past)
        ch = (head[-1] + 1) % 256
        data = head + bytes([ch]) * 5 + bytes([(ch + 7) % 256]) + _tail(20)
        out.append(("close_past%d" % past, data, lv, (nm + past, p + 5)))
    # pieces of 3/4/5/255/256/510/511 bytes that start 2 RLE1 bytes before the cut
    for L in (3, 4, 5, 255, 256, 510, 511):
        p = nm - 2
        head = run_free(p, 30 + L)
        ch = (head[-1] + 1) % 256
        first = min(L, 255)     # the first piece of the run closes the block
        data = head + bytes([ch]) * L + bytes([(ch + 7) % 256]) + _tail(40)
        out.append(("run%d_at_cut" % L, data, lv, (p + _rle(first), p + first)))
    # a run of 255 k + r bytes that the cut falls into
    for r in (0, 1, 4, 254):
        p = nm - 7
        head = run_free(p, 50 + r)
        ch = (head[-1] + 1) % 256
        data = head + bytes([ch]) * (255 * 3 + r) + _tail(60)
        out.append(("run255x3+%d_over_cut" % r, data, lv, (p + 5 + 5, p + 255 + 255)))
    # a full block, then one last piece of 1, 2, 3, 6 or 255 bytes: a block of its own
    for L in (1, 2, 3, 6, 255):
        head = run_free(nm, 70 + L)
        ch = (head[-1] + 1) % 256
        out.append(("last_piece%d" % L, head + bytes([ch]) * L, lv, (nm, nm)))
    # the input ends exactly at a cut: no empty block
    out.append(("ends_at_cut", run_free(nm, 90), lv, (nm, nm)))
    out.append(("ends_at_cut_run", run_free(nm - 5, 91) + b"\x00" * 255, lv, None))
    # all equal
    out.append(("all_equal", b"a" * 300000, lv, None))
    # level 2: a piece right at the cut of a larger block
    head = run_free(nmax(2) - 1, 95)
    out.append(("level2_run4", head + bytes([(head[-1] + 1) % 256]) * 4 + _tail(96), 2, (nmax(2) - 1 + 5, nmax(2) - 1 + 4)))
    # the motivating stream: 99 977 run-free bytes, then a long run
    out.append(("runfree_then_aaaa", motivating(), 1, None))
    return out


def motivating():
    """99 977 run-free bytes and then `a` x 4000: compressjs ends block 1 on four equal bytes without their count byte."""
    head = run_free(99977, 99)
    if head[-1] == ord("a"):
        head = head[:-1] + b"b"
    return head + b"a" * 4000


def check_cut_case(data, level, expect):
    """The case's first block hits the planted corner; the blocks tile the input.  Returns the model's blocks."""
    blocks = M.cut(data, level)
    assert sum(b[1] for b in blocks) == len(data)
    assert all(len(b[2]) >= nmax(level) for b in blocks[:-1])
    assert all(len(b[2]) <= nmax(level) + 4 for b in blocks)
    if expect is not None:
        assert (len(blocks[0][2]), blocks[0][1]) == expect, (len(blocks[0][2]), blocks[0][1], expect)
    return blocks


def _words(n, seed, letters=13):
    rng = np.random.default_rng(seed)
    return b" ".join(bytes(rng.integers(97, 97 + letters, int(l), dtype=np.uint8)) for l in rng.integers(1, 9, n))


def _hit_nmtf(target, seed0):
    """A random block whose zero-run coder output is exactly `target` symbols long (found by search)."""
    for seed in range(seed0, seed0 + 4000):
        rng = np.random.default_rng(seed)
        n = int(target * rng.uniform(0.97, 1.3))
        data = rng.integers(0, 40, n, dtype=np.uint8).tobytes()
        if len(M.mtf_symbols(data)[0]) == target:
            return data
    raise AssertionError("no block with nMTF == %d" % target)


def table_cases():
    """(name, data, level, corner) with corner one of 'nmtf=<k>', 'odd', 'periodic', 'alpha1', 'alpha256'."""
    out = []
    for k, t in enumerate((199, 200, 599, 600, 1199, 1200, 2399, 2400)):
        out.append(("nmtf%d" % t, _hit_nmtf(t, 1000 * k), 1, "nmtf=%d" % t))
    out.append(("alpha1", b"q" * 5000, 1, "alpha1"))
    out.append(("alpha256", bytes(range(256)) * 40, 1, "alpha256"))
    out.append(("words", _words(6000, 7), 1, "odd"))
    for name, d in (("ab_x6000", b"ab" * 6000), ("abc_x3400", b"abc" * 3400), ("aab_x4000", b"aab" * 4000),
                    ("hello_x2500", b"hello" * 2500), ("xyz3", b"xyzxyzxyz")):
        out.append((name, d, 1, "periodic"))
    return out


def check_table_case(data, level, corner):
    """The case reaches its corner in the model."""
    stats = {}
    facts = M.block_facts(data, level, stats)
    if corner.startswith("nmtf="):
        assert facts[0]["m"] == int(corner[5:])
    elif corner == "odd":
        assert stats.get("odd_adjust")
    elif corner == "alpha1":
        assert len(set(data)) == 1
    elif corner == "alpha256":
        assert len(set(data)) == 256
    return facts


def golden_corpus():
    """(key, data, level) of tests/golden/libbz2.json: every cut and table case, the compressjs samples at 1..9, the
    designed table-search blocks of tests/libbz2_table_cases.py (table2_, and all of them as one file) and every case of tests/mtfhuff_cases.py at
    its levels (mtfhuff_; building those needs the oracle)."""
    from tests import libbz2_table_cases as TC
    from tests import mtfhuff_cases as MC
    from tests.util import fixture
    out = [("%s_-%d" % (name, lv), d, lv) for name, d, lv, _ in cut_cases() + table_cases()]
    for i in range(6):
        d = fixture("sample%d.ref" % i)
        out += [("sample%d_-%d" % (i, lv), d, lv) for lv in range(1, 10)]
    out += [("table2_%s_-%d" % (name, lv), d, lv) for name, d, lv in TC.corpus()]
    out.append(("table2_whole_-9", TC.whole(), 9))
    out += [("mtfhuff_%s_-%d" % (c.name, lv), MC.info(c.name).raw, lv) for c in MC.cases() for lv in c.levels]
    return out
