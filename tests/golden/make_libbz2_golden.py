"""Writes tests/golden/libbz2.json: SHA-256 and length of bz2.compress (libbz2 1.0.3 or later) of every input of
tests/libbz2_cases.golden_corpus.  Run from the repository root: python -m tests.golden.make_libbz2_golden"""
import bz2
import hashlib
import json
import os

from tests import libbz2_cases as LC


def main():
    gold = {}
    for key, data, level in LC.golden_corpus():
        z = bz2.compress(data, level)
        gold[key] = {"size": len(z), "sha256": hashlib.sha256(z).hexdigest()}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libbz2.json")
    with open(path, "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
