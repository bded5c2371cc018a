"""The forward-BWT case corpus (tests/bwt_cases.py) reaches every corner it claims, by the CPU model of the path
selection.  tests/test_gpu_bwt_paths.py then holds the GPU to the same model."""
import functools

import numpy as np
import pytest

from tests import bwt_cases as BC


@functools.lru_cache(maxsize=1)
def _models():
    return [BC.Model(c) for c in BC.cases()]


def _names():
    return [c.name for c in BC.cases()]


def test_case_names_are_unique():
    names = _names()
    assert len(names) == len(set(names))


@pytest.mark.parametrize("name", _names())
def test_case_reaches_its_claims(name):
    m = next(m for m in _models() if m.case.name == name)
    assert m.case.claims
    for what, ok in m.case.claims:
        assert ok(m), "%s: %s" % (name, what)
    for batch in (264, 1, 3):
        assert m.margin_ok(batch), "%s: a batch score within 10 %% of 0.5 at %d blocks per batch" % (name, batch)


def test_corpus_reaches_every_finish_and_fallback():
    default = [m.predict() for m in _models()]
    msd_why = direct_why = 0
    for c in default:
        msd_why |= c.bwt_msd_fallback_why
        direct_why |= c.bwt_direct_fallback_why
    assert msd_why == BC.WHY_BUCKET | BC.WHY_CELL | BC.WHY_TIES | BC.WHY_GROUP | BC.WHY_DEPTH
    assert direct_why == BC.WHY_TIES | BC.WHY_GROUP | BC.WHY_DEPTH
    # the LSD direct finish by default (not only with B2_BWT_MSD=0), and each of the others
    assert sum(c.bwt_direct_done for c in default) >= 3
    assert sum(c.bwt_msd_done for c in default) >= 3
    assert sum(c.bwt_wide_batches for c in default) >= 3
    assert sum(c.bwt_rounds_batches - c.bwt_wide_batches for c in default) >= 3
    # every configuration of the GPU matrix runs each finish it can reach somewhere
    for name, (_, cfg) in BC.CONFIGS.items():
        got = [m.predict(**cfg) for m in _models()]
        done = [sum(getattr(c, f) for c in got) for f in ("bwt_msd_done", "bwt_direct_done", "bwt_rounds_batches")]
        assert done[1] > 0 and done[2] > 0 or cfg.get("prefix8"), name
        assert done[0] > 0 or not cfg.get("msd", True) or cfg.get("prefix8"), name


def test_msd_key_is_the_scaled_mixed_radix_number():
    """bwt_msd.cu k_msd_prep: S = floor((2^64 - 1) / a^4), or 2^32 at 256 symbols (the key is the four raw bytes)."""
    g = np.random.default_rng(3)
    for a in (1, 2, 3, 95, 254, 255, 256):
        syms = np.sort(g.permutation(256)[:a]).astype(np.uint8)
        t = syms[g.integers(0, a, size=5000)]
        t[:a] = syms
        hist = np.bincount(t, minlength=256)
        lut = (np.cumsum(hist > 0) - 1).astype(np.int64)
        key = BC.msd_keys(t, a, lut).astype(object)
        n = t.size
        r = [lut[t[(np.arange(n) + j) % n]].astype(object) for j in (1, 2, 3, 4)]
        k = ((r[0] * a + r[1]) * a * a + r[2] * a + r[3])
        S = 1 << 32 if a ** 4 >= 1 << 32 else (2 ** 64 - 1) // a ** 4
        assert list(key) == [(int(x) * S) >> 32 for x in k]
        # order preserving and injective: the cell sort never merges different keys
        order = np.argsort(np.array(k, dtype=np.float64), kind="stable")
        ks = np.array(key, dtype=np.uint64)[order]
        kk = np.array(k, dtype=np.uint64)[order]
        assert np.all((ks[1:] > ks[:-1]) == (kk[1:] > kk[:-1]))
        if a == 256:
            assert list(key) == list(k)
