"""GPU bzip2 decode on the synthetic corpus (tests/synth_corpus.py): streams that reach the corners of the format that
our encoders and libbz2 never write.  Every entry point -- decompressFile, b2_bzip2_decompress_dev, decompressBlock at
every real block, table, and the sharded decode at simulated world sizes 2 and 3 -- must give the writer's expected
bytes, or its error code and nothing else; the oracle must agree with the writer.  The cases aimed at the Huffman
stage run at all three CTA widths of k_hdec, which the decoder picks from the number of block candidates (real
blocks + planted magics)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import bz2synth as W
from tests import synth_corpus as SC

pytestmark = pytest.mark.gpu


def _B():
    from compressjs_b200 import Bzip2
    return Bzip2


def _call(fn):
    from compressjs_b200 import Bzip2Error
    try:
        return ("ok", bytes(fn()))
    except Bzip2Error as e:
        return ("err", e.errorCode)


def _dev(data, exp, multistream=False):
    """b2_bzip2_decompress_dev: device in, device out; on error the output buffer is left alone and out_n is 0."""
    from compressjs_b200 import _native
    L = _native.lib()
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = len(exp[1]) if exp[0] == "ok" else 1 << 16
    out = torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    n = C.c_size_t(12345)
    rc = L.b2_bzip2_decompress_dev(d_in.data_ptr(), d_in.numel(), int(multistream), out.data_ptr(), cap, C.byref(n))
    torch.cuda.synchronize()
    if rc:
        assert n.value == 0 and bool((out == 0xA5).all()), "output written on error"
        return ("err", rc)
    assert bool((out[n.value:] == 0xA5).all()), "written past the decoded length"
    return ("ok", out[:n.value].cpu().numpy().tobytes())


def _sharded(data, world):
    """b2_dec_shard_open/export/finish with `world` simulated ranks: ("ok", bytes) or ("err", code of the earliest error)."""
    from compressjs_b200 import sharded as S, _native
    L = _native.lib()
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    rows = [S.decode_shard_rows(L, d_in, r, world)[1] for r in range(world)]
    all_rows = torch.cat(rows)
    parts, errs, total = [], [], None
    for r in range(world):
        S.decode_shard_rows(L, d_in, r, world)
        o, res = S.decode_shard_finish(L, all_rows, False, d_in.device)
        if o is None:
            errs.append((res["err_idx"], res["err_code"]))
        else:
            parts.append((res["off"], o.cpu().numpy().tobytes()))
            total = res["total"]
    if errs:
        return ("err", min(errs)[1])
    out = b"".join(p for _, p in sorted(parts))
    assert len(out) == total
    return ("ok", out)


def _table(data):
    rows = []
    got = _call(lambda: _B().table(data, lambda p, s: rows.append((p, s))) or b"")
    return got if got[0] == "err" else ("ok", rows)


def _oracle(f, multistream=False):
    from oracle import oracle as O
    try:
        return ("ok", O.bzip2_decompress(f.data, multistream=multistream))
    except O.OracleError as e:
        return ("err", e.errorCode)


def _check_all(f, name):
    exp = f.expect()
    assert _oracle(f) == exp, name
    assert _call(lambda: _B().decompressFile(f.data)) == exp, name
    assert _dev(f.data, exp) == exp, name
    if len(f.members) > 1:
        exp_m = f.expect(True)
        assert _oracle(f, True) == exp_m, name
        assert _call(lambda: _B().decompressFile(f.data, None, True)) == exp_m, name
        assert _dev(f.data, exp_m, True) == exp_m, name
    for pos, b in f.member_blocks[0]:
        e = ("err", b.err) if b.err is not None else (("ok", b.out) if W.crc32(b.out) == b.crc else ("err", W.DATA_ERROR))
        assert _call(lambda: _B().decompressBlock(f.data, pos)) == e, (name, pos)
    assert _table(f.data) == f.expect_table(), name
    for world in (2, 3):
        assert _sharded(f.data, world) == exp, (name, world)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("name", sorted(SC.CASES))
def test_synthetic_case(name):
    c = SC.build(name)
    assert all(c.cond.values()), {k: v for k, v in c.cond.items() if not v}
    if c.hdec:
        assert len(c.file.candidates) <= 2 * _sms()   # k_hdec<512>
    _check_all(c.file, name)


@pytest.mark.parametrize("band", [3, 5])
@pytest.mark.parametrize("name", sorted(n for n in SC.CASES if SC.build(n).hdec))
def test_synthetic_case_hdec_widths(name, band):
    """The same block among tiny filler blocks: 2 x SMs < candidates <= 4 x SMs runs k_hdec<256>, more runs k_hdec<128>."""
    c = SC.build(name)
    m = c.file.members[0]
    filler = W.from_column(b"f", 0, level=m.level)
    k = band * _sms() - len(c.file.candidates)
    f = W.File(W.Member(m.blocks + [filler] * k, m.level))
    cnt, sms = len(f.candidates), _sms()
    assert (2 * sms < cnt <= 4 * sms) if band == 3 else cnt > 4 * sms
    exp = f.expect()
    assert _call(lambda: _B().decompressFile(f.data)) == exp
    assert _dev(f.data, exp) == exp


def test_synthetic_multistream():
    _check_all(SC.multistream_file(), "multistream")


def test_output_past_4gib_on_device():
    """93 maximum-expansion level-9 blocks (46.6 MB each): the decoded stream passes 2^32 bytes."""
    from compressjs_b200 import _native
    b = SC.max_expansion_block()
    assert b.out == b"a" * len(b.out)
    nb = 93
    total = nb * len(b.out)
    assert total > 2 ** 32
    f = W.File(W.Member([b] * nb, 9))
    L = _native.lib()
    d_in = torch.frombuffer(bytearray(f.data), dtype=torch.uint8).cuda()
    out = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    out[total:] = 0xA5
    torch.cuda.synchronize()
    n = C.c_size_t()
    rc = L.b2_bzip2_decompress_dev(d_in.data_ptr(), d_in.numel(), 0, out.data_ptr(), total, C.byref(n))
    torch.cuda.synchronize()
    assert rc == 0, _native.last_error()
    assert n.value == total
    step = 1 << 28
    for s in range(0, total, step):
        assert bool((out[s:min(s + step, total)] == ord("a")).all()), "slice at %d" % s
    assert bool((out[total:] == 0xA5).all())


def test_bound_is_the_only_check_that_fails():
    """A block rejected only by the dbufSize bound of its level decodes, behind a level-9 header, to the bytes its CRC
    was written for: the error the other tests expect can come from nothing but the bound."""
    rel = SC.relevelled()
    assert rel
    for name, f, would_be in rel:
        assert _call(lambda: _B().decompressFile(f.data)) == ("ok", would_be), name
        assert _dev(f.data, ("ok", would_be)) == ("ok", would_be), name
