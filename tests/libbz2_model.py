"""A plain Python model of libbz2's encoder (bzlib 1.0.3 and later): the bytes of ``bz2.compress(data, level)``.

It restates the two stages in which the libbz2 flavor of the GPU encoder differs from the compressjs one -- the RLE1
block cut (runs are never restarted at a block edge; a block holds whole pieces) and the Huffman table search
(``sendMTFValues``: initial partition, four rounds of assign + rebuild, ``BZ2_hbMakeCodeLengths`` with a 17-bit limit)
-- on top of a plain BWT, MTF, zero-run coder and bit packer.  ``cut`` alone is fast enough for inputs of many MB;
``compress`` and ``block_facts`` run the whole model and are meant for inputs of a few hundred KB at most.
"""
import numpy as np


def cut(data, level):
    """The libbz2 blocks of `data`: a list of (raw_start, raw_len, rle1 bytes of the block)."""
    nmax = 100000 * level - 19
    out = []
    i, n = 0, len(data)
    ch, ln = 256, 0          # the pending piece: byte value (256: none) and length
    flushed = 0              # raw bytes in the pieces written so far
    while True:
        blk = bytearray()
        start = flushed

        def piece():
            nonlocal flushed
            if ln < 4:
                blk.extend([ch] * ln)
            else:
                blk.extend([ch] * 4 + [ln - 4])
            flushed += ln
        while i < n and len(blk) < nmax:
            z = data[i]
            i += 1
            if z != ch and ln == 1:
                blk.append(ch)
                flushed += 1
                ch = z
            elif z != ch or ln == 255:
                if ch < 256:
                    piece()
                ch, ln = z, 1
            else:
                ln += 1
        if len(blk) >= nmax:
            out.append((start, flushed - start, bytes(blk)))
            continue
        if ch < 256:
            piece()
            ch, ln = 256, 0
        if blk:
            out.append((start, flushed - start, bytes(blk)))
        return out


def bwt(b):
    """Cyclic BWT, equal rotations in descending start order: (last column, row of rotation 0)."""
    a = np.frombuffer(b, dtype=np.uint8).astype(np.int64)
    n = len(a)
    rank = a.copy()
    h = 1
    while True:
        key2 = np.roll(rank, -h)
        order = np.lexsort((-np.arange(n), key2, rank))
        k = rank[order] * (n + 1) + key2[order]
        newr = np.concatenate(([0], np.cumsum(k[1:] != k[:-1])))
        r2 = np.empty(n, np.int64)
        r2[order] = newr
        rank = r2
        if newr[-1] == n - 1 or h >= n:
            break
        h *= 2
    order = np.lexsort((-np.arange(n), rank))
    return a[(order - 1) % n].astype(np.uint8).tobytes(), int(np.where(order == 0)[0][0])


def mtf_symbols(block):
    """(symbols of the zero-run coder incl. EOB, sorted byte values in use, origPtr)."""
    L, pidx = bwt(block)
    used = sorted(set(block))
    M = list(used)
    syms, run = [], 0
    eob = len(used) + 1

    def flush():
        nonlocal run
        if run:
            z = run - 1
            while True:
                syms.append(1 if z & 1 else 0)
                if z < 2:
                    break
                z = (z - 2) // 2
            run = 0
    for x in L:
        j = M.index(x)
        M.insert(0, M.pop(j))
        if j == 0:
            run += 1
        else:
            flush()
            syms.append(j + 1)
    flush()
    syms.append(eob)
    return syms, used, pidx


def n_groups(nmtf):
    return 2 if nmtf < 200 else 3 if nmtf < 600 else 4 if nmtf < 1200 else 5 if nmtf < 2400 else 6


def make_lengths(freq, max_len=17, stats=None):
    """BZ2_hbMakeCodeLengths.  stats (a dict, optional) counts the 17-bit rescales in 'rescales' and sets 'heap_tie'
    when two equal weights (frequency and depth byte) met at a comparison of the heap."""
    a = len(freq)
    weight, parent, heap = [0] * (2 * a + 2), [0] * (2 * a + 2), [0] * (a + 3)
    for i in range(a):
        weight[i + 1] = (freq[i] if freq[i] else 1) << 8
    while True:
        n_nodes, n_heap = a, 0
        heap[0] = 0
        weight[0] = 0

        def tie(a, b):
            if stats is not None and weight[a] == weight[b]:
                stats["heap_tie"] = True

        def up(z):
            tmp = heap[z]
            tie(tmp, heap[z >> 1])
            while weight[tmp] < weight[heap[z >> 1]]:
                heap[z] = heap[z >> 1]
                z >>= 1
                tie(tmp, heap[z >> 1])
            heap[z] = tmp

        def down(z):
            tmp = heap[z]
            while True:
                y = z << 1
                if y > n_heap:
                    break
                if y < n_heap:
                    tie(heap[y + 1], heap[y])
                    if weight[heap[y + 1]] < weight[heap[y]]:
                        y += 1
                tie(tmp, heap[y])
                if weight[tmp] < weight[heap[y]]:
                    break
                heap[z] = heap[y]
                z = y
            heap[z] = tmp
        for i in range(1, a + 1):
            parent[i] = -1
            n_heap += 1
            heap[n_heap] = i
            up(n_heap)
        while n_heap > 1:
            n1 = heap[1]; heap[1] = heap[n_heap]; n_heap -= 1; down(1)
            n2 = heap[1]; heap[1] = heap[n_heap]; n_heap -= 1; down(1)
            n_nodes += 1
            parent[n1] = parent[n2] = n_nodes
            w1, w2 = weight[n1], weight[n2]
            weight[n_nodes] = ((w1 & ~0xff) + (w2 & ~0xff)) | (1 + max(w1 & 0xff, w2 & 0xff))
            parent[n_nodes] = -1
            n_heap += 1
            heap[n_heap] = n_nodes
            up(n_heap)
        lens, too_long = [], False
        for i in range(1, a + 1):
            j, k = 0, i
            while parent[k] >= 0:
                k = parent[k]
                j += 1
            lens.append(j)
            too_long |= j > max_len
        if not too_long:
            return lens
        if stats is not None:
            stats["rescales"] = stats.get("rescales", 0) + 1
        for i in range(1, a + 1):
            weight[i] = (1 + (weight[i] >> 8) // 2) << 8


def initial_tables(freq, nmtf, ng, report=None):
    """sendMTFValues' initial tables: lists of 0 / 15 lengths; also returns whether the odd-nPart step moved a bound.

    report (a dict, optional) gets 'odd_moved' and 'odd_single': the nPart values at which the odd step moved a bound,
    and at which it was due but skipped because the range was a single symbol; 'exhausted': whether the alphabet ran
    out before nPart reached 1 (the later tables are all 15s); 'ranges': per table the (gs, ge, tFreq) of its part."""
    a = len(freq)
    lens = [[15] * a for _ in range(ng)]
    n_part, rem_f, gs, adjusted = ng, nmtf, 0, False
    moved, single, ranges = [], [], [None] * ng
    while n_part > 0:
        t_freq = rem_f // n_part
        ge, a_freq = gs - 1, 0
        while a_freq < t_freq and ge < a - 1:
            ge += 1
            a_freq += freq[ge]
        odd = n_part != ng and n_part != 1 and (ng - n_part) % 2 == 1
        if ge > gs and odd:
            a_freq -= freq[ge]
            ge -= 1
            adjusted = True
            moved.append(n_part)
        elif ge == gs and odd:
            single.append(n_part)
        ranges[n_part - 1] = (gs, ge, t_freq)
        for v in range(a):
            lens[n_part - 1][v] = 0 if gs <= v <= ge else 15
        n_part -= 1
        gs = ge + 1
        rem_f -= a_freq
    if report is not None:
        report.update(odd_moved=moved, odd_single=single, ranges=ranges,
                      exhausted=any(r[0] > r[1] for r in ranges))
    return lens, adjusted


def tables(syms, alpha_size, stats=None, report=None):
    """(selectors, code lengths of every table) after the four rounds of sendMTFValues.

    report (a dict, optional) gets 'init' (initial_tables' report) and 'rounds': per round a dict of 'ties' (groups
    whose least cost two or more tables share; the first of them is selected), 'max_cost' (the largest cost of a group
    under any table) and 'tables', per table of the round a dict of 'selected' (groups that selected it), 'rescales'
    (17-bit rescales of its build), 'heap_tie', 'max_len' (its longest code) and 'equal_used' (the most used symbols
    that share one frequency in it) and 'zeros' (its symbols of frequency 0, weight 1 in the build).  The tables of round 4 are written."""
    nmtf = len(syms)
    sy = np.asarray(syms, np.int64)
    freq = np.bincount(sy, minlength=alpha_size).tolist()
    ng = n_groups(nmtf)
    init = {}
    lens, adjusted = initial_tables(freq, nmtf, ng, init)
    if stats is not None:
        stats["odd_adjust"] = stats.get("odd_adjust", False) or adjusted
    nsel = (nmtf + 49) // 50
    G = np.zeros((nsel, alpha_size), np.int64)           # symbol counts of every group
    np.add.at(G, (np.arange(nmtf) // 50, sy), 1)
    rounds = []
    for _ in range(4):
        cost = G @ np.array(lens, np.int64).T
        best = cost.min(1)
        sel = np.argmin(cost, axis=1)                    # the first least cost, as the scan of sendMTFValues
        rf = np.zeros((ng, alpha_size), np.int64)
        np.add.at(rf, sel, G)
        built = [{} for _ in range(ng)]
        lens = [make_lengths(rf[t].tolist(), 17, built[t]) for t in range(ng)]
        counts = np.bincount(sel, minlength=ng)
        for t in range(ng):
            f = rf[t][rf[t] > 0]
            if stats is not None:
                stats["rescales"] = stats.get("rescales", 0) + built[t].get("rescales", 0)
            built[t] = dict(selected=int(counts[t]), rescales=built[t].get("rescales", 0),
                            heap_tie=built[t].get("heap_tie", False), max_len=max(lens[t]),
                            equal_used=int(np.bincount(f).max()) if f.size else 0, zeros=int((rf[t] == 0).sum()))
        rounds.append(dict(ties=int(((cost == best[:, None]).sum(1) > 1).sum()), max_cost=int(cost.max()), tables=built))
    if report is not None:
        report.update(init=init, rounds=rounds)
    return sel.tolist(), lens


class _Bits:
    def __init__(self):
        self.parts, self.n = [], 0

    def w(self, n, v):
        self.parts.append(format(v, "0%db" % n))
        self.n += n

    def out(self):
        b = "".join(self.parts)
        b += "0" * (-len(b) % 8)
        return int(b, 2).to_bytes(len(b) // 8, "big") if b else b""


def _crc_table():
    t = []
    for i in range(256):
        c = i << 24
        for _ in range(8):
            c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
        t.append(c)
    return t


_CRC = _crc_table()


def crc32(data, c=0xFFFFFFFF):
    for x in data:
        c = ((c << 8) & 0xFFFFFFFF) ^ _CRC[(c >> 24) ^ x]
    return c ^ 0xFFFFFFFF


def block_facts(data, level, stats=None):
    """Per block what b2_last_trace reports: dicts of raw_start, raw_len, n, m (nMTF), ngroups, nsel."""
    facts = []
    for start, length, blk in cut(data, level):
        syms, _, _ = mtf_symbols(blk)
        if stats is not None:
            tables(syms, len(set(blk)) + 2, stats)
        facts.append(dict(raw_start=start, raw_len=length, n=len(blk), m=len(syms), ngroups=n_groups(len(syms)),
                          nsel=(len(syms) + 49) // 50))
    return facts


TRACE_FIELDS = ("n", "pidx", "m", "alpha", "ngroups", "nsel", "crc", "bit_len")


def encode(data, level):
    """The whole model: (the bytes of bz2.compress(data, level), per block a dict of the TRACE_FIELDS of b2_last_trace
    -- bit_len counts the bits from the block magic to the end of the block's symbols -- together with raw_start,
    raw_len, the zero-run coder's symbols 'syms', the selectors 'sel', the written code lengths 'lens' and the table
    search's 'report' (see tables))."""
    bw = _Bits()
    for ch in b"BZh":
        bw.w(8, ch)
    bw.w(8, ord("0") + level)
    scrc = 0
    blocks = []
    for start, length, blk in cut(data, level):
        b0 = bw.n
        c = crc32(data[start:start + length])
        scrc = (((scrc << 1) | (scrc >> 31)) & 0xFFFFFFFF) ^ c
        bw.w(24, 0x314159); bw.w(24, 0x265359); bw.w(32, c); bw.w(1, 0)
        syms, used, pidx = mtf_symbols(blk)
        bw.w(24, pidx)
        u16 = [any((x >> 4) == i for x in used) for i in range(16)]
        for i in range(16):
            bw.w(1, int(u16[i]))
        uset = set(used)
        for i in range(16):
            if u16[i]:
                for j in range(16):
                    bw.w(1, int((i * 16 + j) in uset))
        a = len(used) + 2
        report = {}
        sel, lens = tables(syms, a, report=report)
        ng = len(lens)
        bw.w(3, ng); bw.w(15, len(sel))
        mt = list(range(ng))
        for s in sel:
            j = mt.index(s)
            mt.insert(0, mt.pop(j))
            bw.w(j + 1, (1 << (j + 1)) - 2)
        codes = []
        for t in range(ng):
            cur = lens[t][0]
            bw.w(5, cur)
            for v in range(a):
                while cur < lens[t][v]:
                    bw.w(2, 2); cur += 1
                while cur > lens[t][v]:
                    bw.w(2, 3); cur -= 1
                bw.w(1, 0)
            code, vec = [0] * a, 0
            for n in range(min(lens[t]), max(lens[t]) + 1):
                for v in range(a):
                    if lens[t][v] == n:
                        code[v] = vec
                        vec += 1
                vec <<= 1
            codes.append(code)
        for gi, g0 in enumerate(range(0, len(syms), 50)):
            ln, cd = lens[sel[gi]], codes[sel[gi]]
            for s in syms[g0:g0 + 50]:
                bw.w(ln[s], cd[s])
        blocks.append(dict(n=len(blk), pidx=pidx, m=len(syms), alpha=len(used), ngroups=ng, nsel=len(sel), crc=c,
                           bit_len=bw.n - b0, raw_start=start, raw_len=length, syms=syms, sel=sel, lens=lens,
                           report=report))
    bw.w(24, 0x177245); bw.w(24, 0x385090); bw.w(32, scrc)
    return bw.out(), blocks


def compress(data, level):
    """The bytes of bz2.compress(data, level)."""
    return encode(data, level)[0]


def trace(data, level):
    """Per block the fields of b2_last_trace (TRACE_FIELDS), as the GPU encoder reports them for the libbz2 flavor."""
    return [tuple(b[f] for f in TRACE_FIELDS) for b in encode(data, level)[1]]
