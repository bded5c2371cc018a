"""The seeded damaged inputs of tests/golden/recover.json (tests/golden/make_recover_golden.py): a spec names the seed,
the size and level of bz2.compress of tests/util.py texty(n, seed), and the damage; build(spec) makes the input."""
import bz2

from tests import recover_model as M
from tests import util as T

SPECS = [
    {"name": "none_l1", "seed": 1, "n": 330000, "level": 1, "damage": ["none"]},
    {"name": "none_l9", "seed": 2, "n": 1200000, "level": 9, "damage": ["none"]},
    {"name": "huffman_flip_b1", "seed": 1, "n": 330000, "level": 1, "damage": ["flip_block", 1, 0.7]},
    {"name": "huffman_flip_b0", "seed": 3, "n": 450000, "level": 1, "damage": ["flip_block", 0, 0.5]},
    {"name": "crc_flip_b2", "seed": 1, "n": 330000, "level": 1, "damage": ["flip_rel", 2, 60]},
    {"name": "zero_inside_b1", "seed": 4, "n": 330000, "level": 1, "damage": ["zero_block", 1, 0.4, 300]},
    {"name": "magic_flip_b2", "seed": 1, "n": 330000, "level": 1, "damage": ["flip_rel", 2, 20]},
    {"name": "eos_flip", "seed": 5, "n": 330000, "level": 1, "damage": ["flip_eos", 10]},
    {"name": "truncated", "seed": 6, "n": 330000, "level": 1, "damage": ["truncate", 0.5]},
    {"name": "two_flips_l2", "seed": 7, "n": 700000, "level": 2, "damage": ["flip_blocks", [0, 2], 0.6]},
]


def _flip(data, bit):
    b = bytearray(data)
    b[bit // 8] ^= 0x80 >> (bit % 8)
    return bytes(b)


def undamaged(spec):
    return bz2.compress(T.texty(spec["n"], spec["seed"]), spec["level"])


def build(spec):
    z = undamaged(spec)
    c = M.candidates(z)
    ends = c[1:] + [_eos(z)]
    kind, *a = spec["damage"]
    if kind == "none":
        return z
    if kind == "flip_block":   # a bit at fraction a[1] of block a[0]'s bits
        k, frac = a
        return _flip(z, c[k] + int((ends[k] - c[k]) * frac))
    if kind == "flip_blocks":
        for k in a[0]:
            z = _flip(z, c[k] + int((ends[k] - c[k]) * a[1]))
        return z
    if kind == "flip_rel":     # a bit at offset a[1] from block a[0]'s magic
        return _flip(z, c[a[0]] + a[1])
    if kind == "flip_eos":
        return _flip(z, _eos(z) + a[0])
    if kind == "zero_block":   # a[2] zero bytes from fraction a[1] of block a[0]
        k, frac, nz = a
        at = (c[k] + int((ends[k] - c[k]) * frac)) // 8
        return z[:at] + bytes(nz) + z[at + nz:]
    if kind == "truncate":     # cut at fraction a[0] of the last block
        return z[:(c[-1] + int((ends[-1] - c[-1]) * a[0])) // 8]
    raise ValueError(kind)


def _eos(z):
    from tests import bz2synth as W
    return W.magic_positions(z)[1][-1]
