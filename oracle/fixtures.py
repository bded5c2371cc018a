"""The compressjs test fixtures (test/sample*) used by the tests and by the benchmark's text workload, rebuilt in
memory from tests/golden/fixtures.xz (see tests/golden/pack_fixtures.py).  Every file is checked against the size
and SHA-256 of the original before it is handed out.
"""
import bz2
import hashlib
import json
import lzma
import os

_GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
_MAN = None
_BLOB = None
_CACHE = {}


def _manifest():
    global _MAN
    if _MAN is None:
        with open(os.path.join(_GOLDEN, "fixtures.json")) as f:
            _MAN = json.load(f)
    return _MAN


def names():
    m = _manifest()
    return sorted(list(m["ref"]) + list(m["bz2"]) + list(m["slice"]) + list(m["text"]))


def _checked(name, b, sig):
    if len(b) != sig["size"] or hashlib.sha256(b).hexdigest() != sig["sha256"]:
        raise RuntimeError("fixture %s does not match its recorded SHA-256" % name)
    return b


def load(name):
    """Bytes of fixture `name` (e.g. "sample4.ref", "sample4.bz2", "sample4.32", "sample4.bzt")."""
    global _BLOB
    if name in _CACHE:
        return _CACHE[name]
    m = _manifest()
    if name in m["ref"]:
        if _BLOB is None:
            with open(os.path.join(_GOLDEN, m["archive"]), "rb") as f:
                _BLOB = lzma.decompress(f.read())
        s = m["ref"][name]
        b = _checked(name, _BLOB[s["offset"]: s["offset"] + s["size"]], s)
    elif name in m["bz2"]:
        s = m["bz2"][name]
        b = _checked(name, bz2.compress(load(s["ref"]), s["level"]), s)
    elif name in m["slice"]:
        s = m["slice"][name]
        b = _checked(name, load(s["ref"])[s["offset"]: s["offset"] + s["size"]], s)
    elif name in m["text"]:
        b = m["text"][name].encode("ascii")
    else:
        raise KeyError("no fixture named %r" % name)
    _CACHE[name] = b
    return b
