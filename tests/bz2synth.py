"""bzip2 streams whose every field is an explicit parameter, for decoder tests (CPU, numpy).

Written from the bzip2 format.  A test can enter at any of four layers:

  content  `from_content(B)`: the block's bytes before RLE1 decode (any bytes, not necessarily valid RLE1 output);
           L and origPtr come from the cyclic BWT (oracle.bwt_cyclic).
  column   `from_column(L, orig)`: any L column and any origPtr, including columns that are not BWT images.
  symbol   `mtf_symbols(L)` gives the MTF + RUNA/RUNB symbols and the used-byte map of a column; `block()` also takes a
           raw symbol list (run digits and EOB anywhere), and `decode_bits()` turns a chosen bit string into the symbols
           that a complete code reads from it (how a magic pattern is planted inside a payload).
  Huffman  `block(...)`: group count, one code-length vector per table (lengths 1-20, any delta path between them),
           the selectors (as table numbers or as raw MTF indices up to groupCount), nSelectors, origPtr, and any
           header field overridden after the fact.

`member()` concatenates blocks at bit granularity behind the 'BZh' + level header and in front of the end-of-stream
magic and the combined stream CRC; `File` concatenates members into a multistream file.

The expected result of every block comes from `model_block`, a plain model of the reference decoder: header checks,
selector MTF over a zero-filled 256-entry list, RUNA/RUNB expansion and inverse MTF with the dbufSize bounds, the
T-vector by a stable counting sort and n steps from origPtr, the reference's RLE1 loop (a byte that follows four equal
bytes is a repeat count) and the bzip2 CRC (polynomial 0x04C11DB7, MSB first).  Every block also reports the
conditions it actually reached (code lengths used, group sizes in bits, selector MTF indices, the inverse-BWT visit
count under the decoder's row sampling, where the RLE1 count bytes sit), so that a test can assert it tested what it
names.
"""
import zlib

import numpy as np

BLOCK_MAGIC = 0x314159265359
EOS_MAGIC = 0x177245385090
GROUP = 50
MAX_LEN = 20
DATA_ERROR, NOT_BZIP, OBSOLETE = -5, -2, -7
IB_STEP = 128          # the GPU inverse BWT walks between rows that are multiples of this (and the start row)
IB_CAP = 512           # bytes one walk records; longer walks are walked again


class ModelError(Exception):
    """A check of the reference decoder fails.  `check` names it when the block still has a defined output with the
    check removed (see `model_block`), None otherwise."""

    def __init__(self, code, what, check=None):
        super().__init__(what)
        self.code, self.check = code, check


# ---- bits ---------------------------------------------------------------------------------------------------------
def bits_of(value, n):
    """n bits of value, MSB first, as a uint8 0/1 array."""
    if n == 0:
        return np.zeros(0, np.uint8)
    return ((int(value) >> np.arange(n - 1, -1, -1, dtype=np.int64)) & 1).astype(np.uint8)


def bits_str(s):
    return np.frombuffer(s.encode(), np.uint8) - ord("0") if s else np.zeros(0, np.uint8)


def pack(bits):
    """0/1 array -> bytes, zero padded to a whole byte."""
    return np.packbits(bits).tobytes()


_REV8 = np.array([int("{:08b}".format(i)[::-1], 2) for i in range(256)], dtype=np.uint8)


def crc32(data):
    """bzip2 CRC-32: polynomial 0x04C11DB7, MSB first.  zlib's CRC-32 is the same code bit-reflected, so it is zlib's
    CRC of the bit-reversed bytes, reversed."""
    a = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data
    r = zlib.crc32(_REV8[a].tobytes())
    return int("{:032b}".format(r)[::-1], 2)


def rotl1(v):
    return ((v << 1) | (v >> 31)) & 0xFFFFFFFF


# ---- codes --------------------------------------------------------------------------------------------------------
def canonical_codes(lens):
    """Code of every symbol: shorter codes first, equal lengths in symbol order (the order a bzip2 decoder's
    limit/base/permute tables assume).  Lengths must satisfy Kraft's inequality (holes are allowed)."""
    lens = [int(x) for x in lens]
    if any(l < 1 or l > MAX_LEN for l in lens):
        raise ValueError("code lengths must be 1..20")
    if sum(1 << (MAX_LEN - l) for l in lens) > 1 << MAX_LEN:
        raise ValueError("over-subscribed code")
    codes = [0] * len(lens)
    code, prev = 0, 0
    for l, s in sorted((l, s) for s, l in enumerate(lens)):
        code <<= l - prev
        codes[s] = code
        code += 1
        prev = l
    return codes


def chain_lengths(nsym, maxlen, order=None):
    """A complete code on nsym symbols whose longest codes have exactly `maxlen` bits: lengths 1, 2, ..., maxlen-1,
    maxlen, maxlen, then the deepest code shorter than maxlen is split until there are nsym codes.  order[k] is the
    symbol that gets the k-th shortest code (default: symbol order)."""
    if nsym < maxlen + 1:
        raise ValueError("a complete code on %d symbols cannot reach %d bits" % (nsym, maxlen))
    ls = list(range(1, maxlen)) + [maxlen, maxlen]
    while len(ls) < nsym:
        k = max(i for i, l in enumerate(ls) if l < maxlen)
        l = ls.pop(k)
        ls[k:k] = [l + 1, l + 1]
    ls.sort()
    order = list(range(nsym)) if order is None else list(order)
    out = [0] * nsym
    for k, s in enumerate(order):
        out[s] = ls[k]
    return out


def uniform_lengths(nsym):
    """Every symbol at ceil(log2(nsym)) bits (a code with holes unless nsym is a power of two)."""
    return [max(1, int(np.ceil(np.log2(nsym))))] * nsym


def decode_bits(bits, lens, avoid=()):
    """The symbols that the code `lens` reads from the bit string `bits` ('0'/'1'), padded with zeros until the last
    code is complete.  Raises ValueError if one of them is in `avoid` (e.g. EOB, or run digits)."""
    codes = canonical_codes(lens)
    table = {(l, c): s for s, (l, c) in enumerate(zip(lens, codes))}
    out, cur, n, i = [], 0, 0, 0
    while i < len(bits) or n:
        cur = (cur << 1) | (int(bits[i]) if i < len(bits) else 0)
        n += 1
        i += 1
        if (n, cur) in table:
            s = table[(n, cur)]
            if s in avoid:
                raise ValueError("bit string decodes to symbol %d" % s)
            out.append(s)
            cur, n = 0, 0
        elif n > MAX_LEN:
            raise ValueError("code has a hole on this bit string")
    return out


# ---- symbol layer -------------------------------------------------------------------------------------------------
def run_digits(r):
    """RUNA (0) / RUNB (1) digits of a run of r >= 1 copies (bijective base 2, least significant digit first)."""
    out = []
    while r > 0:
        if r & 1:
            out.append(0)
            r -= 1
        else:
            out.append(1)
            r -= 2
        r >>= 1
    return out


def mtf_symbols(L, used=None):
    """MTF + RUNA/RUNB symbols of column L over the sorted used-byte list, EOB appended.  Returns (symbols, used)."""
    L = bytes(L)
    used = sorted(set(L)) if used is None else list(used)
    idx = {b: i for i, b in enumerate(used)}
    lst = list(range(len(used)))
    out, run = [], 0
    for b in L:
        s = idx[b]
        if lst[0] == s:
            run += 1
            continue
        if run:
            out += run_digits(run)
            run = 0
        j = lst.index(s)
        del lst[j]
        lst.insert(0, s)
        out.append(j + 1)
    if run:
        out += run_digits(run)
    out.append(len(used) + 1)
    return out, used


def selector_mtf(tables, gc):
    """MTF indices that encode the table sequence `tables` (list starts as 0..gc-1)."""
    lst = list(range(gc))
    out = []
    for t in tables:
        j = lst.index(t)
        del lst[j]
        lst.insert(0, t)
        out.append(j)
    return out


def selectors_from_mtf(mtf, gc):
    """The reference decoder's selector list: MTF over a zero-filled 256-entry list whose first gc slots are 0..gc-1.
    Index gc is legal (it reads a slot behind the tables); above that is a data error."""
    lst = list(range(gc)) + [0] * (256 - gc)
    out = []
    for j in mtf:
        if j > gc:
            raise ModelError(DATA_ERROR, "selector MTF index %d > groupCount" % j)   # no defined output
        v = lst.pop(j)
        lst.insert(0, v)
        out.append(v)
    return out


# ---- decode model -------------------------------------------------------------------------------------------------
def model_unmtf(symbols, used, dbuf, relax=()):
    """RUNA/RUNB expansion and inverse MTF of the reference decoder up to the first EOB.  Returns the L column.
    The dbufSize bounds named in `relax` are skipped."""
    sym_total = len(used)
    lst = list(range(256))
    vals, reps = [], []
    count, run_pos, tt = 0, 0, 0
    for s in symbols:
        if s <= 1:
            if not run_pos:
                run_pos, tt = 1, 0
            tt += run_pos * (s + 1)
            run_pos <<= 1
            continue
        if run_pos:
            run_pos = 0
            if count + tt > dbuf and "run past dbufSize" not in relax:
                raise ModelError(DATA_ERROR, "run past dbufSize", "run past dbufSize")
            vals.append(used[lst[0]] if lst[0] < sym_total else 0)
            reps.append(tt)
            count += tt
        if s > sym_total:
            break
        if count >= dbuf and "literal past dbufSize" not in relax:
            raise ModelError(DATA_ERROR, "literal past dbufSize", "literal past dbufSize")
        v = lst.pop(s - 1)
        lst.insert(0, v)
        vals.append(used[v])
        reps.append(1)
        count += 1
    return np.repeat(np.array(vals, np.uint8), np.array(reps, np.int64))


def model_ibwt(L, orig):
    """T-vector by a stable counting sort of L, then n steps from origPtr.  Returns (B, rows walked, cycle length).
    An origPtr >= n reads an entry of the zero-filled T-vector buffer that the sort did not write: the walk starts at
    row 0."""
    n = L.size
    T = np.argsort(L, kind="stable")
    r0 = int(T[orig]) if orig < n else 0
    Tl = T.tolist()
    cyc = [r0]
    row = Tl[r0]
    while row != r0 and len(cyc) < n:
        cyc.append(row)
        row = Tl[row]
    rows = np.resize(np.array(cyc, np.int64), n)
    return L[rows], rows, len(cyc)


def rle1_classes(B):
    """Positions of the count bytes in B under the reference's RLE1 loop, and whether B ends in an uncounted run of four."""
    n = B.size
    is_count = np.zeros(n, bool)
    if n == 0:
        return is_count, False
    starts = np.flatnonzero(np.r_[True, B[1:] != B[:-1]])
    lens = np.diff(np.r_[starts, n])
    pending = False
    for s, r in zip(starts.tolist(), lens.tolist()):
        if pending:
            is_count[s] = True
            s += 1
            r -= 1
            pending = False
        if r >= 5:
            is_count[s + 4:s + r:5] = True
        if r % 5 == 4:
            pending = True
    return is_count, pending


def model_rle1(B):
    is_count, pending = rle1_classes(B)
    prev = np.r_[np.uint8(0), B[:-1]] if B.size else B
    vals = np.where(is_count, prev, B)
    reps = np.where(is_count, B.astype(np.int64), 1)
    return np.repeat(vals, reps), is_count, pending


def model_block(symbols, used, orig, sel_tables, nsel, level, rand=0, gc=2, hole_at=None, relax=()):
    """Expected output bytes of one block, or ModelError with the reference's error code.  Returns (out, info).

    The checks named in `relax` are skipped, which gives what the block decodes to without them: the symbols after
    nSelectors groups keep the last selector's table (that is how the writer codes them), a code hole is stepped over,
    the dbufSize bounds are not applied, and an origPtr >= n starts the walk at row 0."""
    dbuf = 100000 * level

    def check(name, code=DATA_ERROR):
        if name not in relax:
            raise ModelError(code, name, name)

    if rand:
        check("randomised block", OBSOLETE)
    if orig > dbuf:
        check("origPtr > dbufSize")
    if not 2 <= gc <= 6 or nsel == 0:
        raise ModelError(DATA_ERROR, "groupCount / nSelectors")
    sym_total = len(used)
    eob = next((i for i, s in enumerate(symbols) if s > 1 and s > sym_total), None)
    if eob is None:
        raise ModelError(DATA_ERROR, "no EOB: the decoder reads past the symbols")
    if eob // GROUP >= nsel:
        check("selectors exhausted")
    if hole_at is not None and hole_at <= eob:
        check("code hole")
    L = model_unmtf(symbols[:eob + 1], used, dbuf, relax)
    if orig >= L.size:
        check("origPtr >= block length")
    B, rows, cyc = model_ibwt(L, orig)
    out, is_count, pending = model_rle1(B)
    return out, dict(L=L, B=B, rows=rows, cycle=cyc, is_count=is_count, pending=pending)


# ---- reports ------------------------------------------------------------------------------------------------------
def ibwt_report(rows, n):
    """Visits of the GPU inverse BWT: the walk from the start row is cut at every row that is a multiple of IB_STEP and
    at the start row itself; each piece is one visit."""
    r0 = int(rows[0])
    cut = ((rows & (IB_STEP - 1)) == 0) | (rows == r0)
    at = np.flatnonzero(cut)
    seg = np.diff(np.r_[at, n])
    return dict(visits=int(at.size), max_visit=int(seg.max()) if seg.size else 0, start_row=r0)


def rle1_report(B, is_count, pending):
    pos = np.flatnonzero(is_count)
    val = B[pos]
    n = B.size
    lens = np.where(is_count, B.astype(np.int64), 1)
    tile_out = np.add.reduceat(lens, np.arange(0, n, 2048)) if n else np.zeros(0, np.int64)
    # maximal equal-byte runs of B that hold a count byte equal to the run byte
    eq_runs = set()
    if n:
        starts = np.flatnonzero(np.r_[True, B[1:] != B[:-1]])
        rl = np.diff(np.r_[starts, n])
        cnt_in = np.add.reduceat(is_count.astype(np.int64), starts)
        eq_runs = set(int(x) for x in rl[cnt_in > 0].tolist())
    return dict(
        count_pos=pos, count_val=val,
        count0_mod8=set((pos[val == 0] % 8).tolist()), count255_mod8=set((pos[val == 255] % 8).tolist()),
        count_tile_cross=int(np.count_nonzero((pos - 4) // 2048 != pos // 2048)),
        count_at_tile_edge=set(int(x) for x in val[(pos % 2048) < 4].tolist()),
        max_tile_out=int(tile_out.max()) if tile_out.size else 0,
        last_is_count=bool(n and is_count[-1]), trailing_run4=bool(pending),
        eq_count_runs=eq_runs)


# ---- Huffman layer: one block -------------------------------------------------------------------------------------
class Block:
    """One block: .bits (0/1 array from its magic to behind its last code), .out (expected bytes) or .err (expected
    error code), .crc, .report."""


def block(symbols, used, orig, level=9, lens=None, tables=None, sel_mtf=None, nsel=None, paths=None, tail_bits="",
          hole_at=None, crc=None, rand=0, gc=None, L=None):
    """Write one block.

    symbols  symbol list (RUNA=0, RUNB=1, MTF index j as j+1, EOB = len(used)+1), usually ending in EOB
    used     sorted used bytes (the 16x16 bitmap); symTotal = len(used)
    lens     one code-length list (len(used)+2 entries) per table; default two tables of uniform lengths
    tables   table number of every selector; or sel_mtf: raw selector MTF indices (0..groupCount)
    nsel     nSelectors (default: what the symbols need, padded with selectors that repeat the last table)
    paths    paths[g][i]: lengths the delta code passes through before it settles on lens[g][i]
    tail_bits bits written behind the symbols
    hole_at  in front of symbol hole_at, write the all-ones word of the longest code length of that symbol's table,
             which must be a hole of the code (no code is a prefix of it)
    crc, rand, gc: header fields written as given instead of what the content implies

    A block that fails a check of the decoder still carries the CRC of what it decodes to with the failing check
    removed (`model_block`), so that only that check can make a decoder reject it: .err is the expected error code,
    .failed the checks that fail in decode order, .would_be those bytes.  Only when no such output is defined (no
    EOB, a selector MTF index above groupCount, a bad groupCount or nSelectors) is the CRC 0.
    """
    symbols = [int(s) for s in symbols]
    used = [int(u) for u in used]
    sym_count = len(used) + 2
    if lens is None:
        lens = [uniform_lengths(sym_count)] * 2
    lens = [list(map(int, l)) for l in lens]
    ngroups = len(lens)
    gc_field = ngroups if gc is None else gc
    need = max(1, -(-len(symbols) // GROUP))
    if sel_mtf is None:
        tables = [0] * need if tables is None else list(tables)
        if nsel is None:
            nsel = max(need, len(tables))
        tables = (tables + [tables[-1]] * nsel)[:nsel]
        sel_mtf = selector_mtf(tables, ngroups)
    else:
        sel_mtf = list(sel_mtf)
        if nsel is None:
            nsel = len(sel_mtf)
    R = Block()
    R.level, R.used, R.orig, R.symbols = level, used, orig, symbols
    R.sel_mtf = sel_mtf
    try:
        R.tables = selectors_from_mtf(sel_mtf, ngroups)
    except ModelError as e:
        R.tables = None
        sel_err = e
    R.out, R.err, R.would_be, info, out = None, None, None, None, None
    R.failed = []
    while True:
        try:
            if R.tables is None:
                raise sel_err
            out, info = model_block(symbols, used, orig, R.tables, nsel, level, rand=rand, gc=gc_field, hole_at=hole_at,
                                    relax=R.failed)
            break
        except ModelError as e:
            if R.err is None:
                R.err, R.why = e.code, str(e)
            R.failed.append(e.check or str(e))
            if e.check is None:
                break
    if out is not None:
        if R.err is None:
            R.out = out.tobytes()
        else:
            R.would_be = out.tobytes()
    R.crc = (crc32(out) if out is not None else 0) if crc is None else crc
    codes = [canonical_codes(l) for l in lens]

    parts = [bits_of(BLOCK_MAGIC, 48), bits_of(R.crc, 32), bits_of(rand, 1), bits_of(orig, 24)]
    hi = [any((u >> 4) == k for u in used) for k in range(16)]
    parts.append(np.array(hi, np.uint8))
    for k in range(16):
        if hi[k]:
            parts.append(np.array([(k << 4 | j) in used for j in range(16)], np.uint8))
    parts += [bits_of(gc_field, 3), bits_of(nsel, 15)]
    parts.append(bits_str("".join("1" * j + "0" for j in sel_mtf)))
    # code lengths: 5-bit start, then per symbol +1 ("10") / -1 ("11") steps through the path, "0" to settle.  The
    # report counts full swings: the delta code reaching 1 after 20 or 20 after 1 (a step path is monotone between
    # waypoints, so only waypoints can be extremes)
    R.delta_range, R.delta_swings = [], []
    for g in range(ngroups):
        t = lens[g][0] if not (paths and paths[g] and paths[g][0]) else paths[g][0][0]
        s = ["{:05b}".format(t)]
        lo, hi_, swings, last = t, t, 0, t if t in (1, MAX_LEN) else None
        for i in range(sym_count):
            for w in (list(paths[g][i]) if paths and paths[g] else []) + [lens[g][i]]:
                s.append(("10" if w > t else "11") * abs(w - t))
                t = w
                lo, hi_ = min(lo, t), max(hi_, t)
                if t in (1, MAX_LEN):
                    swings += last is not None and t != last
                    last = t
            s.append("0")
        parts.append(bits_str("".join(s)))
        R.delta_range.append((lo, hi_))
        R.delta_swings.append(int(swings))
    # payload: code of every symbol under its group's table
    sym = np.array(symbols, np.int64)
    if sym.size:
        grp = np.arange(sym.size) // GROUP
        # groups behind the last selector keep its table
        tl = R.tables or [0]
        tabs = np.array((tl + [tl[-1]] * (grp[-1] + 1))[:grp[-1] + 1], np.int64)[grp]
        code_t = np.array(codes, np.int64)
        len_t = np.array(lens, np.int64)
        c, l = code_t[tabs, sym], len_t[tabs, sym]
        sh = l[:, None] - 1 - np.arange(MAX_LEN)[None, :]
        m = sh >= 0
        pay = ((c[:, None] >> np.maximum(sh, 0)) & 1)[m].astype(np.uint8)
        R.hole = None
        if hole_at is not None:
            g = int(tabs[hole_at])
            ml = max(lens[g])
            ones = (1 << ml) - 1
            assert all((k, ones >> (ml - k)) not in set(zip(lens[g], codes[g])) for k in range(1, ml + 1)), "not a hole"
            R.hole = (g, ml)
            pay = np.insert(pay, int(l[:hole_at].sum()), np.ones(ml, np.uint8))
        parts.append(pay)
        gbits = np.add.reduceat(l, np.arange(0, sym.size, GROUP))
        eob = next((i for i, s in enumerate(symbols) if s > 1 and s > len(used)), sym.size - 1)
        R.max_code_len = int(l[:eob + 1].max())
        R.eob_index = eob
        R.group_bits = gbits
    else:
        R.max_code_len, R.group_bits, R.eob_index, R.hole = 0, np.zeros(0, np.int64), None, None
    parts.append(bits_str(tail_bits))
    R.bits = np.concatenate(parts)
    R.lens, R.nsel = lens, nsel
    R.report = {}
    if info is not None:
        R.report.update(n=int(info["L"].size), L=info["L"], B=info["B"], cycle=info["cycle"])
        R.report.update(ibwt_report(info["rows"], info["L"].size))
        R.report.update(rle1_report(info["B"], info["is_count"], info["pending"]))
    if L is not None and info is not None:
        assert np.array_equal(info["L"], np.frombuffer(bytes(L), np.uint8)), "symbols do not rebuild L"
    return R


def from_column(L, orig, used=None, **kw):
    """Column layer: any L column and origPtr."""
    syms, used = mtf_symbols(L, used)
    return block(syms, used, orig, L=L, **kw)


def from_content(B, **kw):
    """Content layer: the block's bytes before RLE1 decode; L and origPtr from the cyclic BWT."""
    from oracle import oracle as O
    L, orig = O.bwt_cyclic(bytes(B))
    return from_column(L, orig, **kw)


# ---- streams ------------------------------------------------------------------------------------------------------
class Member:
    def __init__(self, blocks, level=9, level_byte=None, stream_crc=None):
        self.blocks, self.level = blocks, level
        self.level_byte = ord("0") + level if level_byte is None else level_byte
        scrc = 0
        for b in blocks:
            scrc = rotl1(scrc) ^ b.crc
        self.stream_crc = scrc if stream_crc is None else stream_crc
        self.crc_ok = self.stream_crc == scrc
        parts = [np.unpackbits(np.frombuffer(b"BZh" + bytes([self.level_byte]), np.uint8))]
        self.block_pos = []
        pos = 32
        for b in blocks:
            self.block_pos.append(pos)
            parts.append(b.bits)
            pos += b.bits.size
        self.eos_pos = pos
        parts += [bits_of(EOS_MAGIC, 48), bits_of(self.stream_crc, 32)]
        self.data = pack(np.concatenate(parts))


def magic_positions(data):
    """Bit offsets of every block magic and end-of-stream magic in data (any bit phase)."""
    bits = np.unpackbits(np.frombuffer(data, np.uint8))
    found = {BLOCK_MAGIC: [], EOS_MAGIC: []}
    for ph in range(8):
        sh = np.packbits(bits[ph:]).tobytes()
        for m in found:
            pat = m.to_bytes(6, "big")
            i = sh.find(pat)
            while i >= 0:
                found[m].append(8 * i + ph)
                i = sh.find(pat, i + 1)
    return sorted(found[BLOCK_MAGIC]), sorted(found[EOS_MAGIC])


class File:
    """Members concatenated.  .data, .expect(multistream) -> ('ok', bytes) | ('err', code), .block_starts (absolute bit
    positions of the first member's blocks), .planted_block / .planted_eos (magic patterns that are not stream
    structure), .candidates (every block-magic position: what the GPU decoder has to decode)."""

    def __init__(self, members):
        if isinstance(members, Member):
            members = [members]
        self.members = members
        self.data = b"".join(m.data for m in members)
        self.block_starts, real_eos, off = [], [], 0
        self.member_blocks = []
        for m in members:
            self.member_blocks.append([(off + p, b) for p, b in zip(m.block_pos, m.blocks)])
            self.block_starts += [off + p for p in m.block_pos]
            real_eos.append(off + m.eos_pos)
            off += len(m.data) * 8
        bm, em = magic_positions(self.data)
        self.planted_block = sorted(set(bm) - set(self.block_starts))
        self.planted_eos = sorted(set(em) - set(real_eos))
        self.candidates = bm

    def expect(self, multistream=False):
        out = []
        for m in self.members[: None if multistream else 1]:
            if not 1 <= m.level_byte - ord("0") <= 9:
                return ("err", NOT_BZIP)
            for b in m.blocks:
                if b.err is not None:
                    return ("err", b.err)
                out.append(b.out)
                if crc32(b.out) != b.crc:
                    return ("err", DATA_ERROR)
            if not m.crc_ok:
                return ("err", DATA_ERROR)
        return ("ok", b"".join(out))

    def expect_table(self):
        rows = []
        for pos, b in self.member_blocks[0]:
            if b.err is not None or crc32(b.out) != b.crc:
                return ("err", b.err if b.err is not None else DATA_ERROR)
            rows.append((pos, len(b.out)))
        return ("ok", rows)
