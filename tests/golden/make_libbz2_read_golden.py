"""Generate tests/golden/libbz2_read.json: libbz2's verdict on every case of tests/libbz2_read_cases.py.

The verdict restates bzip2 -d's member loop over bz2.BZ2Decompressor: a member must end (d.eof), and behind it the
remaining bytes, up to four, are compared with "BZh1".."BZh9": nothing left ends the file, a mismatch is trailing
garbage and is ignored, a match of fewer than four bytes is a truncated file, four matching bytes start the next
member.  The golden keeps, per case, the SHA-256 of the input (so drift in the writer is caught), accept or reject, and
on accept the size and SHA-256 of the output.

    python tests/golden/make_libbz2_read_golden.py
"""
import bz2
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests import libbz2_read_cases as LC  # noqa: E402


def libbz2_read(data):
    """(accepted, output) of bzip2 -d on data."""
    out, rest, first = [], data, True
    while True:
        if not first:
            if not rest:
                break
            head = rest[:4]
            if not all(head[k] == b"BZh"[k] if k < 3 else 0x31 <= head[k] <= 0x39 for k in range(len(head))):
                break
            if len(head) < 4:
                return False, b"".join(out)
        d = bz2.BZ2Decompressor()
        try:
            out.append(d.decompress(rest))
        except OSError:
            return False, b"".join(out)
        if not d.eof:
            return False, b"".join(out)
        rest, first = d.unused_data, False
    return True, b"".join(out)


def verdict(data):
    ok, out = libbz2_read(data)
    v = {"input_sha256": hashlib.sha256(data).hexdigest(), "accept": ok}
    if ok:
        v.update(size=len(out), sha256=hashlib.sha256(out).hexdigest())
    return v


def main():
    g = {name: verdict(LC.build(name).data) for name in sorted(LC.CASES)}
    with open(os.path.join(HERE, "libbz2_read.json"), "w") as f:
        json.dump(g, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
