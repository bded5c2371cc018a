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
    """BZ2_hbMakeCodeLengths.  stats (a dict, optional) counts the 17-bit rescales in 'rescales'."""
    a = len(freq)
    weight, parent, heap = [0] * (2 * a + 2), [0] * (2 * a + 2), [0] * (a + 3)
    for i in range(a):
        weight[i + 1] = (freq[i] if freq[i] else 1) << 8
    while True:
        n_nodes, n_heap = a, 0
        heap[0] = 0
        weight[0] = 0

        def up(z):
            tmp = heap[z]
            while weight[tmp] < weight[heap[z >> 1]]:
                heap[z] = heap[z >> 1]
                z >>= 1
            heap[z] = tmp

        def down(z):
            tmp = heap[z]
            while True:
                y = z << 1
                if y > n_heap:
                    break
                if y < n_heap and weight[heap[y + 1]] < weight[heap[y]]:
                    y += 1
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


def initial_tables(freq, nmtf, ng):
    """sendMTFValues' initial tables: lists of 0 / 15 lengths; also returns whether the odd-nPart step moved a bound."""
    a = len(freq)
    lens = [[15] * a for _ in range(ng)]
    n_part, rem_f, gs, adjusted = ng, nmtf, 0, False
    while n_part > 0:
        t_freq = rem_f // n_part
        ge, a_freq = gs - 1, 0
        while a_freq < t_freq and ge < a - 1:
            ge += 1
            a_freq += freq[ge]
        if ge > gs and n_part != ng and n_part != 1 and (ng - n_part) % 2 == 1:
            a_freq -= freq[ge]
            ge -= 1
            adjusted = True
        for v in range(a):
            lens[n_part - 1][v] = 0 if gs <= v <= ge else 15
        n_part -= 1
        gs = ge + 1
        rem_f -= a_freq
    return lens, adjusted


def tables(syms, alpha_size, stats=None):
    """(selectors, code lengths of every table) after the four rounds of sendMTFValues."""
    nmtf = len(syms)
    freq = [0] * alpha_size
    for s in syms:
        freq[s] += 1
    ng = n_groups(nmtf)
    lens, adjusted = initial_tables(freq, nmtf, ng)
    if stats is not None:
        stats["odd_adjust"] = stats.get("odd_adjust", False) or adjusted
    for _ in range(4):
        rf = [[0] * alpha_size for _ in range(ng)]
        sel = []
        for g0 in range(0, nmtf, 50):
            grp = syms[g0:g0 + 50]
            costs = [sum(lens[t][s] for s in grp) for t in range(ng)]
            bt = costs.index(min(costs))
            sel.append(bt)
            for s in grp:
                rf[bt][s] += 1
        lens = [make_lengths(rf[t], 17, stats) for t in range(ng)]
    return sel, lens


class _Bits:
    def __init__(self):
        self.bits = []

    def w(self, n, v):
        for i in range(n - 1, -1, -1):
            self.bits.append((v >> i) & 1)

    def out(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return np.packbits(np.array(b, dtype=np.uint8)).tobytes() if b else b""


def crc32(data, c=0xFFFFFFFF):
    for x in data:
        c ^= x << 24
        for _ in range(8):
            c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
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


def compress(data, level):
    """The whole model: the bytes of bz2.compress(data, level)."""
    bw = _Bits()
    for ch in b"BZh":
        bw.w(8, ch)
    bw.w(8, ord("0") + level)
    scrc = 0
    for start, length, blk in cut(data, level):
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
        sel, lens = tables(syms, a)
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
            t = sel[gi]
            for s in syms[g0:g0 + 50]:
                bw.w(lens[t][s], codes[t][s])
    bw.w(24, 0x177245); bw.w(24, 0x385090); bw.w(32, scrc)
    return bw.out()
