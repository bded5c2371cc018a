"""Packs the compressjs test fixtures (test/sample*) into tests/golden/fixtures.xz + fixtures.json.

Only the .ref inputs are stored.  Every .bz2 fixture is libbz2's output at the level in its header, and every
block extract (sample2.544888, sample4.*) is a slice of its .ref file, so oracle/fixtures.py derives those;
the .bzt tables are small text and go into the manifest.  The manifest keeps the size and SHA-256 of every
original file, and the loader checks each derived file against them.

  python tests/golden/pack_fixtures.py <compressjs checkout>/test
"""
import bz2
import hashlib
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def _sig(b):
    return {"size": len(b), "sha256": hashlib.sha256(b).hexdigest()}


def main(src):
    names = sorted(os.listdir(src))
    refs = [n for n in names if n.startswith("sample") and n.endswith(".ref")]
    data = {n: open(os.path.join(src, n), "rb").read() for n in names if n.startswith("sample")}
    man = {"archive": "fixtures.xz", "ref": {}, "bz2": {}, "slice": {}, "text": {}}
    blob, off = bytearray(), 0
    for n in refs:
        man["ref"][n] = dict(_sig(data[n]), offset=off)
        blob += data[n]
        off += len(data[n])
    for n, b in sorted(data.items()):
        stem, ext = n.split(".", 1)
        ref = data.get(stem + ".ref")
        if ext == "ref":
            continue
        if ext == "bz2":
            level = b[3] - 0x30
            assert ref is not None and bz2.compress(ref, level) == b, "%s is not libbz2 -%d of %s.ref" % (n, level, stem)
            man["bz2"][n] = dict(_sig(b), ref=stem + ".ref", level=level)
        elif ext == "bzt":
            man["text"][n] = b.decode("ascii")
        else:
            at = ref.find(b) if ref is not None else -1
            assert at >= 0, "%s is not a slice of %s.ref" % (n, stem)
            man["slice"][n] = dict(_sig(b), ref=stem + ".ref", offset=at)
    filters = [{"id": lzma.FILTER_LZMA2, "preset": 9 | lzma.PRESET_EXTREME, "lc": 4, "lp": 0, "pb": 0, "dict_size": 1 << 26}]
    with open(os.path.join(HERE, "fixtures.xz"), "wb") as f:
        f.write(lzma.compress(bytes(blob), format=lzma.FORMAT_XZ, filters=filters))
    with open(os.path.join(HERE, "fixtures.json"), "w") as f:
        json.dump(man, f, indent=1, sort_keys=True)
        f.write("\n")
    print("packed %d inputs (%d bytes), %d derived files" % (len(refs), len(blob), len(man["bz2"]) + len(man["slice"]) + len(man["text"])))


if __name__ == "__main__":
    main(sys.argv[1])
