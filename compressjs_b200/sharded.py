"""Block-parallel bzip2 encode over the GPUs of one box (SURVEY.md section 8e).

bzip2 blocks are independent once the RLE1 stage has cut them, so every rank encodes a contiguous
range of blocks on its own GPU with no data-path collective.  The only exchange is the final
bitstream gather (north_star: "NCCL over NVLink only for the final bitstream gather"):

  1. every rank cuts the blocks (b2_bzip2_plan -- a cheap scan) and encodes blocks
     [first, first+count) into a fragment that starts at bit 0 of a private buffer
     (b2_bzip2_encode_range_dev)
  2. all_gather of (fragment bits, block count)   -> every rank knows its global bit offset
  3. the fragment is shifted to (global offset mod 8) so that only whole bytes move
  4. the byte fragments travel to rank 0 straight into their final place in the output buffer
     (NCCL send/recv into offset views; no padded staging, no second copy); neighbouring fragments
     share at most one byte, which is OR-ed from the two edge bytes that ride along with the sizes;
     rank 0 adds "BZh"+level and the trailer (stream CRC combined from the per-rank folds of the
     block CRCs, lib/Bzip2.js:917,925-927)

With a sharded INPUT (compress_shares) a rank holds only its share of the bytes plus a halo: the ranks
exchange tiny share summaries (RLE1 run state, leading run, RLE1 output) so that every rank knows the
run state and the RLE1 output in front of its share, cuts its blocks speculatively and checks that the
pieces chain up (b2_bzip2_share_summary / b2_bzip2_plan_share).  The libbz2 flavor's cuts drift away from
multiples of blockSize, so there every rank cuts its share once for every drift its first block can have
(b2_bzip2_share_cut_table), the ranks exchange these tables, and every rank chains them the same way
(libbz2_share_chain) to find the entry of its share.

The resulting stream is byte-identical to Bzip2.compressFile on one GPU (and to the oracle).
The shifting / merging below is plain torch tensor code so that the same logic runs on CPU tensors
with the gloo backend in the unit tests (tests/test_sharded_host.py), where the per-range encoder
is injected.
"""
import ctypes as C
import functools
import time
from collections import namedtuple

import numpy as np

import torch
import torch.distributed as dist

PHASES = {}   # wall-clock milliseconds of the last compress_file_sharded call per phase (rank local)


def _tick(name, t0):
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    t1 = time.perf_counter()
    PHASES[name] = PHASES.get(name, 0.0) + (t1 - t0) * 1e3
    return t1

SQRTPI = 0x177245385090


def block_range(nblocks, rank, world):
    first = rank * nblocks // world
    last = (rank + 1) * nblocks // world
    return first, last - first


def shift_right_bits(frag, nbits, phase):
    """Returns a uint8 tensor holding `frag`'s first nbits starting at bit `phase` (MSB first)."""
    nbytes = (phase + nbits + 7) // 8
    if frag.is_cuda and nbits:
        from . import _native
        out = torch.empty(((phase + nbits + 31) // 32) * 4, dtype=torch.uint8, device=frag.device)
        torch.cuda.current_stream().synchronize()
        rc = _native.lib().b2_bitshift_dev(frag.data_ptr(), nbits, phase, out.data_ptr())
        if rc:
            raise RuntimeError("b2_bitshift_dev: " + _native.last_error())
        return out[:nbytes]
    src = frag[: (nbits + 7) // 8]
    out = torch.zeros(nbytes, dtype=torch.uint8, device=frag.device)
    if nbits == 0:
        return out
    if phase == 0:
        out[: src.numel()] = src
    else:
        s16 = src.to(torch.int16)
        out[: src.numel()] |= (s16 >> phase).to(torch.uint8)
        spill = ((s16 << (8 - phase)) & 0xFF).to(torch.uint8)
        k = min(nbytes - 1, src.numel())
        out[1: 1 + k] |= spill[:k]
    # clear the bits behind the fragment
    tail = (phase + nbits) % 8
    if tail:
        out[-1] &= (0xFF << (8 - tail)) & 0xFF
    return out


def fold_stream_crc(crcs):
    s = 0
    for c in crcs:
        s = (((s << 1) | (s >> 31)) ^ int(c)) & 0xFFFFFFFF  # lib/Bzip2.js:917
    return s


def trailer_bytes(bitpos, stream_crc):
    """The 80 trailer bits placed at absolute bit `bitpos`: (first byte index, bytes)."""
    val = (SQRTPI << 32) | stream_crc
    phase = bitpos % 8
    total = phase + 80
    nbytes = (total + 7) // 8
    val <<= nbytes * 8 - total
    return bitpos // 8, val.to_bytes(nbytes, "big")


def assemble(level, frags, bits, crcs_per_rank, device):
    """Rank-0 side: frags[r] = byte tensor already shifted to its phase; bits[r] = fragment bits."""
    offs, o = [], 32
    for b in bits:
        offs.append(o)
        o += int(b)
    total_bits = o + 80
    nbytes_out = (total_bits + 7) // 8
    out = torch.empty(nbytes_out, dtype=torch.uint8, device=device)
    out[max(0, nbytes_out - 12):] = 0   # trailer region (OR-ed below)
    out[:4] = torch.tensor(list(b"BZh" + bytes([0x30 + level])), dtype=torch.uint8, device=device)
    edge = {}                   # bytes shared by two neighbours: byte index -> OR of the contributions
    for r, f in enumerate(frags):
        if bits[r] == 0:
            continue
        b0 = offs[r] // 8
        nb = (offs[r] % 8 + int(bits[r]) + 7) // 8
        if nb > 2:
            out[b0 + 1: b0 + nb - 1] = f[1: nb - 1].to(device)     # interior bytes belong to this fragment alone
        for bi in {0, nb - 1}:
            edge[b0 + bi] = edge.get(b0 + bi, 0) | int(f[bi])
    for k, v in edge.items():
        if k >= 4:
            out[k] = v
    crcs = [c for rc in crcs_per_rank for c in rc]
    b0, tb = trailer_bytes(o, fold_stream_crc(crcs))
    # the first trailer byte may share its byte with the last fragment (already written via `edge`)
    out[b0: b0 + len(tb)] |= torch.tensor(list(tb), dtype=torch.uint8, device=device)
    return out


def rotl32(v, k):
    k %= 32
    return ((v << k) | (v >> (32 - k))) & 0xFFFFFFFF if k else v & 0xFFFFFFFF


class SharedHostBuffer:
    """A page-locked host buffer that all ranks of one box map (POSIX shared memory, registered with CUDA in every
    process): every GPU downloads its fragment over its own PCIe link straight to its final place in the stream."""

    def __init__(self, nbytes, group=None):
        from multiprocessing import shared_memory, resource_tracker
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        names = [None]
        if rank == 0:
            self.shm = shared_memory.SharedMemory(create=True, size=max(int(nbytes), 4096))
            names = [self.shm.name]
        if dist.is_initialized():
            dist.broadcast_object_list(names, src=0, group=group)
        if rank != 0:
            self.shm = shared_memory.SharedMemory(name=names[0])
            try:  # only the creator unlinks the segment
                resource_tracker.unregister(self.shm._name, "shared_memory")
            except Exception:
                pass
        self.owner = rank == 0
        self.tensor = torch.frombuffer(self.shm.buf, dtype=torch.uint8)
        self.registered = False
        if torch.cuda.is_available():
            rc = torch.cuda.cudart().cudaHostRegister(self.tensor.data_ptr(), self.tensor.numel(), 0)
            self.registered = int(rc) == 0

    def close(self):
        if self.registered:
            torch.cuda.cudart().cudaHostUnregister(self.tensor.data_ptr())
            self.registered = False
        self.tensor = None
        try:
            self.shm.close()
            if self.owner:
                self.shm.unlink()
        except Exception:
            pass


def place_fragments(frag, nbits, count, crcs, level, device, group=None, host_out=None, keep_sharded=False):
    """Every rank contributes a fragment (uint8 tensor starting at bit 0, nbits long) with `count` blocks and their
    CRCs; returns the complete .bz2 stream on rank 0 (None elsewhere).  The interior bytes of every fragment are
    received directly at their final byte offset of the output.  With host_out (a SharedHostBuffer's tensor, the same
    memory on every rank) the stream is assembled in host memory instead: every rank downloads its own fragment into
    place and rank 0 gets the stream's length back.  With keep_sharded nothing moves: every rank gets a ShardedStream
    (its piece at its final bit position; .gather() finishes the job when one GPU wants the whole stream)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    t0 = time.perf_counter()
    if world == 1:
        return assemble(level, [frag], [nbits], [crcs], device)
    # 1. sizes, block counts and the fold of the own block CRCs (lib/Bzip2.js:917 is linear: folds combine by rotation)
    mine = torch.tensor([nbits, count, fold_stream_crc(crcs)], dtype=torch.int64, device=device)
    allv = [torch.zeros(3, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(allv, mine, group=group)
    meta = [[int(x) for x in v.tolist()] for v in allv]
    bits = [m[0] for m in meta]
    offs, o = [], 32
    for b in bits:
        offs.append(o)
        o += b
    total_bits = o + 80
    phase = offs[rank] % 8
    t0 = _tick("allgather_sizes", t0)
    shifted = shift_right_bits(frag, nbits, phase)
    nb = (phase + nbits + 7) // 8 if nbits else 0
    t0 = _tick("shift", t0)
    # 2. the two edge bytes of every fragment (they may share their byte with a neighbour)
    eb = torch.zeros(2, dtype=torch.uint8, device=device)
    if nb:
        eb[0] = shifted[0]
        eb[1] = shifted[nb - 1]
    alle = [torch.zeros(2, dtype=torch.uint8, device=device) for _ in range(world)]
    dist.all_gather(alle, eb, group=group)
    nbs = [((offs[r] % 8) + bits[r] + 7) // 8 if bits[r] else 0 for r in range(world)]
    if host_out is not None:
        # 3'. interiors: every GPU writes its own piece of the host buffer (parallel PCIe links), then a barrier
        if nb > 2:
            b0 = offs[rank] // 8
            host_out[b0 + 1: b0 + nb - 1].copy_(shifted[1: nb - 1], non_blocking=True)
            if shifted.is_cuda:
                torch.cuda.current_stream().synchronize()
        dist.barrier(group=group)
        t0 = _tick("d2h_place", t0)
        if rank != 0:
            return None
        hb = host_out.numpy()
        for r in range(world):
            if nbs[r]:
                b0 = offs[r] // 8
                e0, e1 = int(alle[r][0]), int(alle[r][1])
                if r == 0 or (offs[r] % 8) == 0:
                    hb[b0] = e0
                else:
                    hb[b0] |= e0
                if nbs[r] > 1:
                    hb[b0 + nbs[r] - 1] = e1
        scrc = 0
        for m in meta:
            scrc = rotl32(scrc, m[1]) ^ m[2]
        b0t, tb = trailer_bytes(o, scrc)
        first_shared = (o % 8) != 0
        for k, v in enumerate(tb):
            if k == 0 and first_shared:
                hb[b0t] |= v
            else:
                hb[b0t + k] = v
        hb[:4] = np.frombuffer(b"BZh" + bytes([0x30 + level]), dtype=np.uint8)
        _tick("edges_trailer", t0)
        return (total_bits + 7) // 8
    st = ShardedStream(shifted, nb, offs, nbs, alle, meta, o, total_bits, level, rank, world, group, device)
    if keep_sharded:
        return st
    return st.gather()


class ShardedStream:
    """The finished stream, left where it was produced: every rank holds its fragment already shifted to its final bit
    position (`piece`, whose byte 0 is byte `offset` of the stream; neighbours share at most their edge bytes, which
    combine by OR) and everything needed to finish it (edge bytes of all fragments, block counts and CRC folds).
    gather() moves the pieces to rank 0 and returns the complete .bz2 there."""

    def __init__(self, shifted, nb, offs, nbs, alle, meta, o, total_bits, level, rank, world, group, device):
        self.piece, self.nb, self.offs, self.nbs, self.alle, self.meta = shifted, nb, offs, nbs, alle, meta
        self.end_bit, self.total_bits, self.level = o, total_bits, level
        self.rank, self.world, self.group, self.device = rank, world, group, device
        self.offset = offs[rank] // 8
        self.total_bytes = (total_bits + 7) // 8

    def _fixups(self):
        """Header, shared edge bytes and trailer: {byte offset: value} (the same on every rank)."""
        edge = {}
        for r in range(self.world):
            if self.nbs[r]:
                b0 = self.offs[r] // 8
                e0, e1 = int(self.alle[r][0]), int(self.alle[r][1])
                edge[b0] = edge.get(b0, 0) | e0
                edge[b0 + self.nbs[r] - 1] = edge.get(b0 + self.nbs[r] - 1, 0) | e1
        scrc = 0
        for m in self.meta:
            scrc = rotl32(scrc, m[1]) ^ m[2]
        b0t, tb = trailer_bytes(self.end_bit, scrc)
        fix = {b0t + k: v for k, v in enumerate(tb)}
        for k, v in edge.items():
            if k >= 4:
                fix[k] = fix.get(k, 0) | v
        for k, v in enumerate(b"BZh" + bytes([0x30 + self.level])):
            fix[k] = v
        return fix

    def write_file(self, path):
        """Every rank writes the interior bytes of its piece at their offset of `path` (one file, visible to all ranks);
        rank 0 sizes the file first and adds the header, the bytes neighbours share and the trailer.  Returns the
        stream length.  The consumer-side counterpart of leaving the stream sharded: no rank ever holds the whole file."""
        import os
        if self.rank == 0:
            with open(path, "wb") as f:
                f.truncate(self.total_bytes)
        if self.world > 1:
            dist.barrier(group=self.group)
        fd = os.open(path, os.O_WRONLY)
        try:
            if self.nb > 2:
                os.pwrite(fd, self.piece[1: self.nb - 1].cpu().numpy().tobytes(), self.offset + 1)
            if self.rank == 0:
                for k, v in sorted(self._fixups().items()):
                    os.pwrite(fd, bytes([v]), k)
        finally:
            os.close(fd)
        if self.world > 1:
            dist.barrier(group=self.group)
        return self.total_bytes

    def gather(self):
        rank, world, group, device = self.rank, self.world, self.group, self.device
        shifted, nb, offs, nbs, alle, meta, o = self.piece, self.nb, self.offs, self.nbs, self.alle, self.meta, self.end_bit
        t0 = time.perf_counter()
        # 3. interiors: point to point into the output
        ops, out = [], None
        if rank == 0:
            out = torch.empty(self.total_bytes, dtype=torch.uint8, device=device)
            for r in range(1, world):
                if nbs[r] > 2:
                    b0 = offs[r] // 8
                    ops.append(dist.P2POp(dist.irecv, out[b0 + 1: b0 + nbs[r] - 1], r, group))
            if nbs[0] > 2:
                b0 = offs[0] // 8
                out[b0 + 1: b0 + nbs[0] - 1] = shifted[1: nbs[0] - 1]
        elif nb > 2:
            ops.append(dist.P2POp(dist.isend, shifted[1: nb - 1].contiguous(), 0, group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        t0 = _tick("p2p_place", t0)
        if rank != 0:
            return None
        # 4. header, edge bytes, trailer
        fix = self._fixups()
        idx = torch.tensor(list(fix.keys()), dtype=torch.int64, device=device)
        val = torch.tensor(list(fix.values()), dtype=torch.uint8, device=device)
        out[idx] = val
        _tick("edges_trailer", t0)
        return out


def compress_sharded(encode_range, nblocks, level, device, group=None):
    """encode_range(first, count) -> (uint8 tensor fragment starting at bit 0, nbits, [block crcs]).
    Returns the complete .bz2 stream as a uint8 tensor on rank 0 (None elsewhere)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    first, count = block_range(nblocks, rank, world)
    t0 = time.perf_counter()
    frag, nbits, crcs = encode_range(first, count)
    _tick("encode_range", t0)
    return place_fragments(frag, nbits, count, crcs, level, device, group)


FLAVORS = {"compressjs": 0, "libbz2": 1}   # B2_BZ2_COMPRESSJS, B2_BZ2_LIBBZ2


def _flavor_id(flavor):
    if flavor not in FLAVORS:
        raise ValueError("unknown bzip2 flavor %r (expected 'compressjs' or 'libbz2')" % (flavor,))
    return FLAVORS[flavor]


def _range_encoder(L, d_in, n, level, flavor="compressjs"):
    from . import _native
    fl = _flavor_id(flavor)

    def encode_range(first, count):
        if count == 0:
            return torch.zeros(8, dtype=torch.uint8, device=d_in.device), 0, []
        cap = count * 1400000 + 4096
        out = torch.empty(cap, dtype=torch.uint8, device=d_in.device)
        bits = C.c_uint64()
        crcs = (C.c_uint32 * count)()
        rc = L.b2_bzip2_encode_range_dev_flavor(d_in.data_ptr(), n, level, first, count, 0, out.data_ptr(), cap, C.byref(bits), crcs, fl)
        if rc:
            raise RuntimeError("b2_bzip2_encode_range_dev_flavor: " + _native.last_error())
        return out, int(bits.value), list(crcs)

    return encode_range


def gpu_encode_range_fn(d_in, level, flavor="compressjs"):
    """encode_range callable backed by libb2bz.so for a uint8 CUDA tensor holding the whole input
    (exact plan: every block boundary of the file is cut on this GPU)."""
    from . import _native
    L = _native.lib()
    n = d_in.numel()
    fl = _flavor_id(flavor)
    total = C.c_size_t()
    rc = L.b2_bzip2_plan_flavor(d_in.data_ptr(), n, level, C.byref(total), fl)
    if rc:
        raise RuntimeError("b2_bzip2_plan_flavor: " + _native.last_error())
    return _range_encoder(L, d_in, n, level, flavor), int(total.value)


def spec_plan_ok(infos, n):
    """infos[r] = (raw_start, raw_end, first, planned, cut, total) of every rank's speculative plan."""
    world = len(infos)
    total = infos[0][5]
    pos = 0
    nxt = 0
    for r in range(world):
        s, e, first, planned, cut, tot = infos[r]
        if tot != total or first != nxt or cut != planned:
            return False
        if planned:
            if s != pos:
                return False
            pos = e
        nxt = first + planned
    return nxt == total and pos == n


def compress_file_sharded(d_in, level=9, group=None, flavor="compressjs"):
    """Whole-file bzip2 encode of a CUDA uint8 tensor present on every rank; stream on rank 0.

    Block cutting: every rank cuts only ITS share of the blocks from a speculative start boundary
    (b2_bzip2_plan_spec); the ranks then check that the pieces chain exactly (end(r) == start(r+1), ...).
    If a run-phase slip makes the speculation fail anywhere, all ranks fall back to the exact plan.
    flavor="libbz2" writes the bytes of libbz2 (bz2.compress): its cuts drift away from multiples of blockSize,
    so every rank takes the exact plan of the whole input and encodes its range of the blocks."""
    from . import _native
    L = _native.lib()
    n = d_in.numel()
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if world == 1 or _flavor_id(flavor) != FLAVORS["compressjs"]:
        enc, nblocks = gpu_encode_range_fn(d_in, level, flavor)
        return compress_sharded(enc, nblocks, level, d_in.device, group)
    PHASES.clear()
    t0 = time.perf_counter()
    info = (C.c_uint64 * 6)()
    rc = L.b2_bzip2_plan_spec(d_in.data_ptr(), n, level, rank, world, info)
    if rc:
        raise RuntimeError("b2_bzip2_plan_spec: " + _native.last_error())
    mine = torch.tensor([int(v) for v in info], dtype=torch.int64, device=d_in.device)
    allv = [torch.zeros(6, dtype=torch.int64, device=d_in.device) for _ in range(world)]
    dist.all_gather(allv, mine, group=group)
    infos = [tuple(int(x) for x in v.tolist()) for v in allv]
    _tick("plan_spec+verify", t0)
    if spec_plan_ok(infos, n):
        enc = _range_encoder(L, d_in, n, level)
        first, count = infos[rank][2], infos[rank][3]
        return compress_sharded(lambda f, c: enc(first, count), infos[0][5], level, d_in.device, group)
    enc, nblocks = gpu_encode_range_fn(d_in, level)
    return compress_sharded(enc, nblocks, level, d_in.device, group)


# ---- sharded input ---------------------------------------------------------------------------------
# Host mirror of the RLE1 scan state of csrc/rle1.cu (rs_make / rs_combine): bit 63 non-empty, bit 62 "one run",
# first byte << 24, last byte << 16, trailing run length mod 255 << 8, length mod 255.
def outfresh(c):
    """RLE1 bytes produced by c bytes of one run consumed from a fresh state (lib/Bzip2.js:636-667)."""
    q, r = divmod(c, 255)
    return 5 * q + (r if r <= 3 else 5)


def rs_combine(A, B):
    if not (A >> 63):
        return B
    if not (B >> 63):
        return A
    a_all, b_all = (A >> 62) & 1, (B >> 62) & 1
    a_fc, a_lc, a_tr, a_len = (A >> 24) & 255, (A >> 16) & 255, (A >> 8) & 255, A & 255
    b_fc, b_lc, b_tr, b_len = (B >> 24) & 255, (B >> 16) & 255, (B >> 8) & 255, B & 255
    join = a_lc == b_fc
    trail = (a_tr + b_len) % 255 if (b_all and join) else b_tr
    return (1 << 63) | ((a_all & b_all & int(join)) << 62) | (a_fc << 24) | (b_lc << 16) | (trail << 8) | ((a_len + b_len) % 255)


def share_plan_inputs(summaries, level):
    """summaries[r] = (state, lead, w_fresh, n) of rank r's share (b2_bzip2_share_summary), in rank order.
    Returns ([(state_in, w_in, first, count, raw_offset)] per rank, total blocks, total RLE1 bytes).
    A block belongs to the rank in whose share it starts: block k starts behind the byte that completes k * blockSize
    RLE1 bytes (if no run-phase slip happened before it -- the ranks verify that afterwards)."""
    BS = level * 100000 - 19
    st, W, g = 0, 0, 0
    ins = []
    for (state, lead, w_fresh, n) in summaries:
        ins.append((st, W, g))
        if n:
            c = ((st >> 8) & 255) if (st >> 63) and ((st >> 16) & 255) == ((state >> 24) & 255) else 0
            W += outfresh(c + lead) - outfresh(c) + (w_fresh - outfresh(lead))
            st = rs_combine(st, state)
            g += n
    total = (W + BS - 1) // BS

    def before(w):      # blocks that start at or before the raw position whose RLE1 prefix is w
        return 0 if w == 0 else min(total, w // BS + 1)
    firsts = [before(w) for (_, w, _) in ins] + [total]
    res = []
    for r, (st_in, w_in, g0) in enumerate(ins):
        n = summaries[r][3]
        first = firsts[r]
        count = (firsts[r + 1] - first) if n else 0
        res.append((st_in, w_in, first, count, g0))
    return res, total, W


CUT_NOT_PIECE, CUT_STEP_EXACT, CUT_BUF_END = 1, 2, 4   # flags of a cut-table row (include/b2bz.h B2_CUT_*)


def share_drift_bound(w_in, level):
    """The largest drift the first block of a share that starts at W position w_in can have: 4 per block in front."""
    M = level * 100000 - 19
    return 4 * ((w_in + M - 1) // M)


def libbz2_share_chain(ins, w_total, tables, level, ends_input):
    """Chains the libbz2 cut tables of all shares, in rank order.  ins = share_plan_inputs(...)[0]; w_total = RLE1 bytes
    of the whole input; tables[r] = rank r's rows indexed by entry drift, (k, blocks, exit drift, flags) as
    b2_bzip2_share_cut_table writes them (a [drifts, 4] array or a list of rows; None for an empty share); ends_input[r]: rank r's buffer ends the input.
    Rank 0 enters at block 0 with drift 0 and every rank's row gives the next rank's entry.  Returns
    ([(first block, drift, block count)] per rank, total blocks), or None when some rank's halo is too short for its
    last block (or a row contradicts its entry, which a correct table never does)."""
    M = level * 100000 - 19
    k, d, done = 0, 0, w_total == 0
    res = []
    for r, row_in in enumerate(ins):
        w_in = row_in[1]
        w_end = ins[r + 1][1] if r + 1 < len(ins) else w_total
        if done or k * M + d >= w_end:    # no block starts in this share: the entry passes through
            res.append((k, d, 0))
            continue
        rows = tables[r]
        if rows is None or d >= len(rows):
            return None
        rk, cnt, ex, fl = (int(x) for x in rows[d])
        if rk == k and not (fl & CUT_NOT_PIECE):
            pass
        elif rk + 1 == k and (fl & CUT_STEP_EXACT):   # the entry is within 4 of w_in: row d less its first block
            cnt -= 1
        else:
            return None
        res.append((k, d, cnt))
        if fl & CUT_BUF_END:
            if not ends_input[r]:
                return None
            done = True
            k += cnt
        else:
            k, d = k + cnt, ex
    if not done:
        return None
    return res, k


def _i64(v):
    return v - (1 << 64) if v >= (1 << 63) else v


def _u64(v):
    return v + (1 << 64) if v < 0 else v


def _all_gather_tables(rows, ends_input, world, group, dev):
    """All-gather of every rank's cut table (an int32 array [drifts, 4]) and of whether its buffer ends the input.  The
    tables differ in length: the ranks first exchange (rows, ends flag), then their tables padded to the longest one, so
    each rank receives world x 16 x (rows of the longest table) bytes.  Returns ([int32 numpy array per rank], [flags])."""
    if world == 1:
        return [rows], [ends_input]
    head = torch.tensor([rows.shape[0], int(ends_input)], dtype=torch.int64, device=dev)
    heads = [torch.zeros_like(head) for _ in range(world)]
    dist.all_gather(heads, head, group=group)
    heads = [v.tolist() for v in heads]
    pad = torch.zeros((max(h[0] for h in heads) or 1, 4), dtype=torch.int32, device=dev)
    pad[: rows.shape[0]] = torch.from_numpy(rows).to(dev)
    allp = [torch.zeros_like(pad) for _ in range(world)]
    dist.all_gather(allp, pad, group=group)
    return [allp[r][: heads[r][0]].cpu().numpy() for r in range(world)], [bool(h[1]) for h in heads]


def _gpu_share_cut_table(L, d_buf, share_len, level, st_in, w_in, dmax):
    """b2_bzip2_share_cut_table: rows (k, blocks, exit drift, flags) for the entry drifts 0..dmax, as an int32 numpy
    array [dmax + 1, 4] (every field is below 2^31: block indices and drifts of inputs under 50 TB)."""
    from . import _native
    tab = (C.c_uint32 * (4 * (dmax + 1)))()
    rc = L.b2_bzip2_share_cut_table(d_buf.data_ptr(), d_buf.numel(), level, st_in, w_in, share_len, dmax, tab)
    if rc:
        raise RuntimeError("b2_bzip2_share_cut_table: " + _native.last_error())
    return np.frombuffer(tab, dtype=np.int32).reshape(-1, 4).copy()


def _gpu_plan_share(L, d_buf, level, st_in, w_in, first, count, drift, flavor):
    from . import _native
    info = (C.c_uint64 * 6)()
    rc = L.b2_bzip2_plan_share_flavor(d_buf.data_ptr(), d_buf.numel(), level, st_in, w_in, first, count, drift, _flavor_id(flavor), info)
    if rc:
        raise RuntimeError("b2_bzip2_plan_share_flavor: " + _native.last_error())
    return [int(v) for v in info]


def compress_shares(d_buf, share_len, level=9, group=None, host_out=None, keep_sharded=False, flavor="compressjs"):
    """Whole-file bzip2 encode when every rank holds only ITS share of the input: d_buf = CUDA uint8 tensor with the
    share (share_len bytes) followed by a halo (the first bytes of the next shares; empty on the last rank).  The shares
    are contiguous in rank order.  Returns the stream on rank 0 (None elsewhere); with keep_sharded a ShardedStream on
    every rank (the output stays sharded like the input; .gather() assembles it on rank 0).
    flavor="libbz2" writes the bytes of libbz2 (bz2.compress): every rank cuts its share for every drift its first
    block can have, the tables are all-gathered (16 bytes per drift, 4 drifts per block in front of the share, every
    table padded to the longest) and chained the same way on every rank.  A halo too short for a share's last block falls back to the whole input."""
    from . import _native
    L = _native.lib()
    libbz2 = _flavor_id(flavor) == FLAVORS["libbz2"]
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    dev = d_buf.device
    PHASES.clear()
    if d_buf.is_cuda:
        torch.cuda.current_stream().synchronize()   # the library works on its own stream: the input must have landed
    t0 = time.perf_counter()
    summ = (C.c_uint64 * 4)()
    rc = L.b2_bzip2_share_summary(d_buf.data_ptr(), share_len, summ)
    if rc:
        raise RuntimeError("b2_bzip2_share_summary: " + _native.last_error())
    mine = torch.tensor([_i64(int(v)) for v in summ], dtype=torch.int64, device=dev)
    if world > 1:
        allv = [torch.zeros(4, dtype=torch.int64, device=dev) for _ in range(world)]
        dist.all_gather(allv, mine, group=group)
    else:
        allv = [mine]
    summaries = [tuple(_u64(int(x)) for x in v.tolist()) for v in allv]
    plan, total, w_total = share_plan_inputs(summaries, level)
    st_in, w_in, first, count, g0 = plan[rank]
    n_total = sum(sm[3] for sm in summaries)
    t0 = _tick("share_summaries", t0)
    drift, chain = 0, None
    if libbz2:
        # every rank's cut for every entry drift; all ranks chain the same tables to the same entries
        if share_len:
            rows = _gpu_share_cut_table(L, d_buf, share_len, level, st_in, w_in, share_drift_bound(w_in, level))
        else:
            rows = np.zeros((0, 4), dtype=np.int32)
        t0 = _tick("cut_table", t0)
        alltab, ends = _all_gather_tables(rows, g0 + d_buf.numel() == n_total, world, group, dev)
        tables = [alltab[r] if summaries[r][3] else None for r in range(world)]
        chain = libbz2_share_chain(plan, w_total, tables, level, ends)
        t0 = _tick("cut_table_exchange", t0)
        if chain is not None:
            (first, drift, count), total = chain[0][rank], chain[1]
    row = [0, 0, first, count, 0, 0]
    if chain is not None or not libbz2:
        row = _gpu_plan_share(L, d_buf, level, st_in, w_in, first, count, drift, flavor)
    mine = torch.tensor([row[0] + g0, row[1] + g0, row[2], row[3], row[4], total], dtype=torch.int64, device=dev)
    if world > 1:
        alli = [torch.zeros(6, dtype=torch.int64, device=dev) for _ in range(world)]
        dist.all_gather(alli, mine, group=group)
    else:
        alli = [mine]
    infos = [tuple(int(x) for x in v.tolist()) for v in alli]
    _tick("plan_share+verify", t0)
    if (libbz2 and chain is None) or not spec_plan_ok(infos, n_total):
        # a run-phase slip or a block longer than the halo: every rank gets the whole input and the exact plan decides
        PHASES["fallback_full_input"] = 1.0
        lens = [sm[3] for sm in summaries]
        parts = [torch.empty(max(ln, 1), dtype=torch.uint8, device=dev) for ln in lens]
        maxlen = max(lens + [1])
        pad = torch.zeros(maxlen, dtype=torch.uint8, device=dev)
        pad[:share_len] = d_buf[:share_len]
        if world > 1:
            gl = [torch.empty(maxlen, dtype=torch.uint8, device=dev) for _ in range(world)]
            dist.all_gather(gl, pad, group=group)
            full = torch.cat([gl[r][: lens[r]] for r in range(world)])
        else:
            full = d_buf[:share_len]
        del parts
        return compress_file_sharded(full, level, group, flavor)
    t0 = time.perf_counter()
    enc = _range_encoder(L, d_buf, d_buf.numel(), level, flavor)
    frag, nbits, crcs = enc(first, count)
    _tick("encode_range", t0)
    return place_fragments(frag, nbits, count, crcs, level, dev, group, host_out, keep_sharded)


def share_bounds(n, rank, world, halo):
    """Equal contiguous shares of n bytes: (first byte, share length, bytes to hold = share + halo)."""
    g0 = rank * n // world
    g1 = (rank + 1) * n // world
    return g0, g1 - g0, min(n, g1 + halo) - g0


# ---- sharded decode -------------------------------------------------------------------------------
def decode_shard_rows(L, d_in, rank, world, flavor="compressjs"):
    """Stage 1 on one rank: returns (info, rows) -- rows = int64 tensor [own candidates, 6] on the CPU.  The session
    reads in `flavor` until its finish."""
    from . import _native
    fl = _flavor_id(flavor)
    if d_in.is_cuda:
        torch.cuda.current_stream().synchronize()   # the library works on its own stream: the input must have landed
    info = (C.c_uint64 * 3)()
    rc = L.b2_dec_shard_open_flavor(d_in.data_ptr(), d_in.numel(), rank, world, info, fl)
    if rc:
        raise RuntimeError("b2_dec_shard_open: %s (code %d)" % (_native.last_error(), rc))
    total, lo, hi = int(info[0]), int(info[1]), int(info[2])
    buf = (C.c_uint64 * (6 * max(hi - lo, 1)))()
    rc = L.b2_dec_shard_export(buf)
    if rc:
        raise RuntimeError("b2_dec_shard_export: " + _native.last_error())
    rows = torch.tensor([int(v) if int(v) < 2 ** 63 else int(v) - 2 ** 64 for v in buf[: 6 * (hi - lo)]], dtype=torch.int64).reshape(-1, 6)
    return (total, lo, hi), rows


def decode_shard_finish(L, all_rows, multistream, device, flavor="compressjs"):
    """Stage 2 on one rank: all_rows = [total candidates, 6] int64 (CPU).  Returns (own output tensor, res).  The
    session finishes in the flavor it was opened with, which `flavor` names."""
    from . import _native
    _flavor_id(flavor)
    flat = [int(v) & (2 ** 64 - 1) for v in all_rows.reshape(-1).tolist()]
    arr = (C.c_uint64 * max(len(flat), 1))(*flat)
    res = (C.c_uint64 * 5)()
    need = 0
    for r in all_rows.tolist():
        need += r[4] if r[0] == 0 else 0
    out = torch.empty(max(need, 1), dtype=torch.uint8, device=device)   # upper bound: everything decodable
    rc = L.b2_dec_shard_finish(arr, int(bool(multistream)), out.data_ptr(), out.numel(), res)
    vals = [int(v) for v in res]
    err_idx = vals[3] if vals[3] < 2 ** 63 else vals[3] - 2 ** 64
    err_code = vals[4] if vals[4] < 2 ** 63 else vals[4] - 2 ** 64
    msg = _native.last_error() if rc else ""
    return out[: vals[1]] if rc == 0 else None, dict(off=vals[0], len=vals[1], total=vals[2], err_idx=err_idx if rc else -1,
                                                      err_code=err_code if rc else 0, msg=msg)


def _decode_whole_input(d_in, multistream=False, group=None, flavor="compressjs"):
    """The sharded decode of a stream held on every rank, up to the error exchange: (own output tensor or None, res) on
    every rank, as decode_shard_finish returns them."""
    from . import _native
    fl = _flavor_id(flavor)
    L = _native.lib()
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    device = d_in.device
    (total, lo, hi), rows = decode_shard_rows(L, d_in, rank, world, flavor)
    if world > 1:
        # every rank scanned the same stream: the candidate counts must agree (a cheap guard against mismatched collectives)
        chk = torch.tensor([total, d_in.numel(), fl], dtype=torch.int64, device=device)
        allc = [torch.zeros_like(chk) for _ in range(world)]
        dist.all_gather(allc, chk, group=group)
        _same_flavor([int(v[2]) for v in allc], "decompress_file_sharded")
        if any(int(v[0]) != total or int(v[1]) != d_in.numel() for v in allc):
            raise RuntimeError("decompress_file_sharded: the ranks do not hold the same stream")
        per = max((r + 1) * total // world - r * total // world for r in range(world))
        pad = torch.zeros((max(per, 1), 6), dtype=torch.int64, device=device)
        if hi > lo:
            pad[: hi - lo] = rows.to(device)
        allp = [torch.zeros_like(pad) for _ in range(world)]
        dist.all_gather(allp, pad, group=group)
        parts = []
        for r in range(world):
            cnt = (r + 1) * total // world - r * total // world
            parts.append(allp[r][:cnt].cpu())
        all_rows = torch.cat(parts) if parts else rows
    else:
        all_rows = rows
    return decode_shard_finish(L, all_rows, multistream, device, flavor)


def _same_flavor(ids, call):
    """Every rank's flavor id, from an exchange: ranks that read in different flavors raise together."""
    if len(set(ids)) > 1:
        names = {v: k for k, v in FLAVORS.items()}
        raise ValueError("%s: the ranks ask for different flavors (%s)" % (call, ", ".join(names.get(i, str(i)) for i in ids)))


def _settle(res, device, group=None):
    """The earliest failing event over all ranks wins (every rank sees the same event list): every rank raises its code,
    with the message on the rank that found it and "Data error" elsewhere.  Otherwise returns every rank's (offset,
    length) of its output in the decoded stream, and the stream's length."""
    from .bzip2 import Bzip2Error
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    mine = torch.tensor([res["err_idx"] if res["err_idx"] >= 0 else 2 ** 62, res["err_code"], res["off"], res["len"], res["total"]],
                        dtype=torch.int64, device=device)
    if world > 1:
        allv = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(allv, mine, group=group)
    else:
        allv = [mine]
    errs = [(int(v[0]), int(v[1]), r) for r, v in enumerate(allv) if int(v[0]) < 2 ** 62]
    if errs:
        idx, code, who = min(errs)
        raise Bzip2Error(code, res["msg"] if who == rank else "Data error")
    return [(int(v[2]), int(v[3])) for v in allv], int(allv[0][4])


def _place(out, spans, total, device, group=None):
    """Every rank's decoded piece travels to rank 0 straight into its place in the decoded stream (send/recv into offset
    views).  Returns the stream on rank 0, None elsewhere."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    ops, full = [], None
    if rank == 0:
        full = torch.empty(total, dtype=torch.uint8, device=device)
        o0, l0 = spans[0]
        full[o0: o0 + l0] = out[:l0]
        for r in range(1, world):
            o, ln = spans[r]
            if ln:
                ops.append(dist.P2POp(dist.irecv, full[o: o + ln], r, group))
    elif out.numel():
        ops.append(dist.P2POp(dist.isend, out.contiguous(), 0, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return full


def decompress_file_sharded(d_in, multistream=False, group=None, flavor="compressjs"):
    """Decode a .bz2 stream held on every rank; the decoded bytes are gathered on rank 0 (uint8 tensor).  flavor as
    Bzip2.decompressFile's: "libbz2" reads as bzip2 -d does.  Every rank must ask for the same flavor."""
    _flavor_id(flavor)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    out, res = _decode_whole_input(d_in, multistream, group, flavor)
    spans, total = _settle(res, d_in.device, group)
    if world == 1:
        return out
    return _place(out, spans, total, d_in.device, group)


# ---- sharded decode from sharded input ------------------------------------------------------------------------------
# A block that decodes to at most 900 000 bytes has at most 900 001 codes of at most 20 bits, at most 32 767 selectors
# and 6 code length tables: with code lengths reached by direct delta paths, about 2.3 MB.  So a block that starts in a
# share ends inside a halo of 4 MiB, the halo compress_shares takes, unless it is corrupt or a table takes a
# pathological delta path; decompress_shares falls back to the whole input then.
DEC_HALO = 4 << 20
DEC_HALO_MIN = 14   # B2_SHARE_HALO_MIN: a magic and its CRC (10 bytes), and the member header behind an end-of-stream magic
SHARE_ROW = 11      # B2_SHARE_ROW: uint64 per exported row (include/b2bz.h)

DecodedShare = namedtuple("DecodedShare", "piece offset total")
DecodedShare.__doc__ = """A rank's piece of the decoded stream: its bytes `piece` are bytes [offset, offset + len(piece)) of
the decoded stream of `total` bytes.  The pieces of all ranks tile the stream."""


def share_layout(sizes):
    """sizes[r] = (share_len, hold) of rank r, in rank order.  Returns (the first byte of every rank's share, the stream's
    length).  Raises ValueError for the first rank whose buffer is not a share of the stream or whose halo is shorter
    than DEC_HALO_MIN bytes and does not reach the stream's end."""
    total = sum(s for s, _ in sizes)
    g0s, g = [], 0
    for r, (share_len, hold) in enumerate(sizes):
        if share_len < 0 or hold < share_len or g + hold > total:
            raise ValueError("decompress_shares: rank %d holds %d bytes from byte %d of a %d-byte stream for a share of %d bytes"
                             % (r, hold, g, total, share_len))
        if g + hold < total and hold - share_len < DEC_HALO_MIN:
            raise ValueError("decompress_shares: rank %d has a halo of %d bytes; a halo must hold at least %d bytes unless it "
                             "reaches the end of the stream" % (r, hold - share_len, DEC_HALO_MIN))
        g0s.append(g)
        g += share_len
    return g0s, total


def _share_open(d_buf, share_len, g0, total, flavor="compressjs"):
    """Stage 1 on one rank (b2_dec_share_open_flavor + export): (rows, 0, "") with rows an int64 CPU tensor [k,
    SHARE_ROW], or (no rows, error code, message) when the open failed, which the caller reports after the exchange.
    The session reads in `flavor` until its finish."""
    from . import _native
    fl = _flavor_id(flavor)
    L = _native.lib()
    if d_buf.is_cuda:
        torch.cuda.current_stream().synchronize()   # the library works on its own stream: the input must have landed
    none = torch.zeros((0, SHARE_ROW), dtype=torch.int64)
    info = (C.c_uint64 * 3)()
    rc = L.b2_dec_share_open_flavor(d_buf.data_ptr(), d_buf.numel(), g0, share_len, total, info, fl)
    if rc:
        return none, rc, "b2_dec_share_open: " + _native.last_error()
    k = int(info[0])
    buf = (C.c_uint64 * (SHARE_ROW * max(k, 1)))()
    rc = L.b2_dec_share_export(buf)
    if rc:
        return none, rc, "b2_dec_share_export: " + _native.last_error()
    rows = np.frombuffer(buf, dtype=np.int64, count=SHARE_ROW * k).reshape(k, SHARE_ROW)
    return torch.from_numpy(rows.copy()), 0, ""


def _share_finish(all_rows, own_rows, multistream, device, flavor="compressjs"):
    """Stage 2 on one rank (b2_dec_share_finish): all_rows = every rank's rows in rank order, own_rows = this rank's.
    Returns (own output tensor, or None on an error, res) with res as decode_shard_finish's plus `unsettled`.  The
    session finishes in the flavor it was opened with, which `flavor` names."""
    from . import _native
    _flavor_id(flavor)
    L = _native.lib()
    flat = np.ascontiguousarray(all_rows.numpy(), dtype=np.int64)
    own = own_rows.numpy()
    need = int(own[(own[:, 1] == 1) & (own[:, 3] == 0), 7].sum())   # upper bound: every owned block that decoded
    out = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    res = (C.c_uint64 * 6)()
    rc = L.b2_dec_share_finish(flat.ctypes.data, flat.shape[0], int(bool(multistream)), out.data_ptr(), out.numel(), res)
    vals = [_i64(int(v)) for v in res]
    msg = _native.last_error() if rc else ""
    err_idx = (vals[3] if vals[3] >= 0 else 0) if rc else -1   # a failure that is no event of the stream fails every rank
    return out[: vals[1]] if rc == 0 else None, dict(off=vals[0], len=vals[1], total=vals[2], err_idx=err_idx,
                                                      err_code=(vals[4] or rc) if rc else 0, msg=msg, unsettled=rc == 0 and vals[5] != 0)


def _gather_shares(d_buf, share_len, lens, group=None):
    """The whole stream on every rank, from every rank's share (lens[r]: rank r's share length)."""
    world = len(lens)
    if world == 1:
        return d_buf[:share_len]
    pad = torch.zeros(max(lens + [1]), dtype=torch.uint8, device=d_buf.device)
    pad[:share_len] = d_buf[:share_len]
    gl = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(gl, pad, group=group)
    return torch.cat([gl[r][: lens[r]] for r in range(world)])


def decompress_shares(d_buf, share_len, multistream=False, group=None, keep_sharded=False, flavor="compressjs"):
    """Decode a .bz2 stream that no rank holds whole: the decode counterpart of compress_shares.  d_buf = uint8 tensor
    with the rank's share of the stream (share_len bytes) followed by a halo, the first bytes of the next shares (at least
    DEC_HALO_MIN bytes unless it reaches the end of the stream; DEC_HALO is enough for any intact block).  The shares are
    contiguous in rank order.  Every rank scans and decodes only the blocks that start in its share; the ranks exchange
    the results, and every rank walks the block chain over all of them.  When the rows cannot settle the stream (a block
    that runs past its owner's halo), every rank gathers the shares and decodes the whole input (decompress_file_sharded's
    path) instead.  The decoded bytes, or the error, are exactly those of Bzip2.decompressFile(stream, multistream=...)
    on one GPU; nothing is delivered on an error.  Returns the decoded stream on rank 0 (None elsewhere); with
    keep_sharded a DecodedShare on every rank (with one rank: the whole stream).  flavor as Bzip2.decompressFile's
    ("libbz2": the result is that of decompressFile(..., flavor="libbz2"), bzip2 -d's); every rank must ask for the same
    one, or all raise ValueError."""
    _flavor_id(flavor)
    stages = [functools.partial(f, flavor=flavor) for f in (_share_open, _share_finish, _decode_whole_input)]
    return _decompress_shares(d_buf, share_len, multistream, group, keep_sharded, *stages, flavor=flavor)


def _decompress_shares(d_buf, share_len, multistream, group, keep_sharded, open_stage, finish_stage, whole_stage, flavor="compressjs"):
    """decompress_shares with its library stages passed in: open_stage(d_buf, share_len, g0, total) -> (rows, code,
    message); finish_stage(all rows, own rows, multistream, device) -> (own output, res); whole_stage(stream,
    multistream, group) -> (own output, res) from the whole input on every rank.  The stages read in `flavor` (bound into
    them by the caller); it travels with the first exchange, so that ranks that ask for different flavors all raise."""
    fl = _flavor_id(flavor)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    dev = d_buf.device
    PHASES.clear()
    # 1. every rank's (share length, bytes held, flavor): where the shares start, the stream's length, every rank's halo
    mine = torch.tensor([share_len, d_buf.numel(), fl], dtype=torch.int64, device=dev)
    if world > 1:
        alls = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(alls, mine, group=group)
    else:
        alls = [mine]
    _same_flavor([int(v[2]) for v in alls], "decompress_shares")
    sizes = [(int(v[0]), int(v[1])) for v in alls]
    g0s, total = share_layout(sizes)
    # 2. open and export; a failed open travels with the row counts, so that every rank raises after the exchange
    rows, rc, msg = open_stage(d_buf, share_len, g0s[rank], total)
    head = torch.tensor([rows.shape[0], rc], dtype=torch.int64, device=dev)
    if world > 1:
        heads = [torch.zeros_like(head) for _ in range(world)]
        dist.all_gather(heads, head, group=group)
    else:
        heads = [head]
    heads = [(int(v[0]), int(v[1])) for v in heads]
    failed = [r for r, (_, code) in enumerate(heads) if code]
    if failed:
        raise RuntimeError(msg if rc else "decompress_shares: rank %d could not open its share (code %d)" % (failed[0], heads[failed[0]][1]))
    # 3. every rank's rows, padded to the longest
    if world > 1:
        pad = torch.zeros((max(k for k, _ in heads) or 1, SHARE_ROW), dtype=torch.int64, device=dev)
        pad[: rows.shape[0]] = rows.to(dev)
        allp = [torch.zeros_like(pad) for _ in range(world)]
        dist.all_gather(allp, pad, group=group)
        all_rows = torch.cat([allp[r][: heads[r][0]].cpu() for r in range(world)])
    else:
        all_rows = rows
    # 4. the walk: every rank sees the same rows, so every rank settles the stream or falls back with the others
    out, res = finish_stage(all_rows, rows, multistream, dev)
    if res["unsettled"]:
        PHASES["fallback_full_input"] = 1.0
        out, res = whole_stage(_gather_shares(d_buf, share_len, [s for s, _ in sizes], group), multistream, group)
    spans, n_out = _settle(res, dev, group)
    if keep_sharded:
        return DecodedShare(out, spans[rank][0], n_out)
    if world == 1:
        return out
    return _place(out, spans, n_out, dev, group)
