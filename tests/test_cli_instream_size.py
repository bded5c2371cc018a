"""The command line's input stream has the reference's `size` (bin/compressjs makeInStream): fstat's size for a regular,
non-empty file, and no attribute for a pipe or an empty file, so that BWTC writes "size unknown" for those."""
import os

from compressjs_b200 import cli


def test_in_stream_size(tmp_path):
    f = tmp_path / "f"
    f.write_bytes(b"abc" * 1000)
    with open(f, "rb") as h:
        assert cli.InStream(h.fileno()).size == 3000
    e = tmp_path / "e"
    e.write_bytes(b"")
    with open(e, "rb") as h:
        assert not hasattr(cli.InStream(h.fileno()), "size")
    r, w = os.pipe()
    os.write(w, b"piped" * 100)
    os.close(w)
    try:
        s = cli.InStream(r)
        assert not hasattr(s, "size")
        assert s.readByte() == ord("p")
    finally:
        os.close(r)
