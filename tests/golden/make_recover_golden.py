"""Generate tests/golden/recover.json: what bzip2recover and libbz2 make of seeded damaged .bz2 files.

Each case is rebuilt from its seed: bz2.compress of tests/util.py texty(n, seed) at `level`, then `damage`.  The golden
keeps the SHA-256 of the damaged input, so drift in either is caught, and for each case bzip2recover's block ranges (the
bits it reports, "block k runs from s to e": s is 48 bits behind the block's magic) and, for each of its rec*.bz2 files
in order, whether bz2.decompress accepts it and the SHA-256 of the bytes it gives.  bzip2recover runs here only:
tests/test_recover_model.py reads the golden.

    python tests/golden/make_recover_golden.py
"""
import bz2
import glob
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests import recover_golden_cases as G  # noqa: E402


def run_bzip2recover(data):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "in.bz2")
        with open(p, "wb") as f:
            f.write(data)
        r = subprocess.run(["bzip2recover", p], capture_output=True, text=True, cwd=d)
        ranges = [[int(a), int(b)] for a, b in re.findall(r"block \d+ runs from (\d+) to (\d+)", r.stderr + r.stdout)]
        files = []
        for q in sorted(glob.glob(os.path.join(d, "rec*in.bz2"))):
            with open(q, "rb") as f:
                z = f.read()
            try:
                files.append({"ok": True, "sha256": hashlib.sha256(bz2.decompress(z)).hexdigest()})
            except (OSError, ValueError, EOFError):
                files.append({"ok": False, "sha256": None})
        return ranges, files


def main():
    out = []
    for spec in G.SPECS:
        data = G.build(spec)
        ranges, files = run_bzip2recover(data)
        out.append(dict(spec, sha256=hashlib.sha256(data).hexdigest(), ranges=ranges, files=files))
    with open(os.path.join(HERE, "recover.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
