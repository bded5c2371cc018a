"""The compressjs command line (bin/compressjs) for the compressors this package has: ``python -m compressjs_b200``.

    python -m compressjs_b200 -z -t bzip2 -9 < file > file.bz2
    python -m compressjs_b200 -d -t bzip2 file.bz2 file

Options, rules and messages are those of bin/compressjs:1-58.  What differs is the choice of compressor: -t takes
``bzip2`` (or ``bzip``) and ``bwtc``; the reference's other compressors, including its default lzp3 (what an absent -t
means), fail with a message instead of writing something the user did not ask for.

As in the reference, BWTC writes the input's size into its header when ``fstat`` of the input gives a non-zero size
(a regular file), and "size unknown" otherwise (a pipe, an empty file): bin/compressjs:60-65 with lib/Util.js:119-124.
The reference writes its output through a 4096-byte buffer that is flushed only when the next byte arrives, and
nothing flushes it when a decode throws (bin/compressjs:103-115): so on a decode error the output holds the bytes
decoded before the error, cut down to a multiple of 4096.

Without -b the command line is a pipe filter for both compressors, as the reference is: the input is read a chunk at a
time and the output written as the library produces it (InStream / OutStream, the makeInStream / makeOutStream of
bin/compressjs:60-120), so memory does not grow with the stream (include/b2bz.h gives the bounds).  -b (the reference
seeks in its input) reads the whole input first.

``-d -t bzip2 --recover`` writes the decoded bytes of every intact block of a damaged file, and ``-d -t bzip2 --repair``
one bzip2 stream made of those blocks (Bzip2.recover).  Both are pipe filters; stderr gets one line per lost block and
a count, and the exit status is 1 when a block was lost.  The output is complete either way.

``-d -t bzip2 --libbz2-decode`` reads .bz2 files as ``bzip2 -d`` does (Bzip2.decompressFile with flavor="libbz2"): every
member, randomised blocks, trailing garbage ignored, and "Unexpected input EOF" for a truncated file.

Usage errors are found before the GPU library is loaded, so they work on a machine without a GPU.
"""
import math
import mmap
import os
import stat
import sys

VERSION = "0.0.1"  # main.js:5

HELP = """
  Usage: python -m compressjs_b200 -d|-z [infile] [outfile]

  Options:

    -h, --help        output usage information
    -V, --version     output the version number
    -d, --decompress  Decompress stdin to stdout
    -z, --compress    Compress stdin to stdout
    -b, --block <n>   Extract a single block, starting at <n> bits.
    -t <compressor>   Select compressor type (bzip2 or bwtc)
    --libbz2          With -z -t bzip2: write the bytes bzip2 (libbz2) writes
    --recover         With -d -t bzip2: write the bytes of every intact block of a damaged file
    --repair          With -d -t bzip2: write one bzip2 stream of every intact block of a damaged file
    --libbz2-decode   With -d -t bzip2: read every member as bzip2 -d (libbz2) reads it
    -1                Fastest/largest compression
    -2
    -3
    -4
    -5
    -6
    -7
    -8
    -9                Slowest/smallest compression

  If <infile> is omitted, reads from stdin.
  If <outfile> is omitted, writes to stdout.
"""

# the compressors of bin/compressjs:133-156 that this package does not have
OTHER_COMPRESSORS = ("defsum", "fenwick", "mtf", "context1", "no", "huff", "huffman", "dmc", "lzjb", "lzjbr", "lzp3",
                     "ppm", "simple")
FLUSH = 4096  # bin/compressjs:103-115


class UsageError(Exception):
    pass


def _number(s):
    """JavaScript's unary + on an option string (NaN for anything that is not a number)."""
    s = s.strip()
    if not s:
        return 0.0
    try:
        return float(int(s, 0)) if s[:2].lower() in ("0x", "0o", "0b") else float(s)
    except ValueError:
        return math.nan


def parse(argv):
    """Returns a dict of the options, or raises UsageError.  --help and --version are returned as 'help'/'version'."""
    opts = {"decompress": False, "compress": False, "block": "-1", "T": None, "levels": set(), "args": [], "libbz2": False,
            "recover": False, "repair": False, "libbz2-decode": False}
    i = 0
    only_args = False
    while i < len(argv):
        a = argv[i]
        i += 1
        if only_args or a == "-" or not a.startswith("-"):
            opts["args"].append(a)
            continue
        if a == "--":
            only_args = True
            continue
        if a.startswith("--"):
            name, eq, val = a[2:].partition("=")
            if name in ("help", "version"):
                return {name: True}
            if name in ("decompress", "compress", "libbz2", "recover", "repair", "libbz2-decode") and not eq:
                opts[name] = True
            elif name == "block":
                if not eq:
                    if i >= len(argv):
                        raise UsageError("error: option `-b, --block <n>' argument missing")
                    val = argv[i]
                    i += 1
                opts["block"] = val
            else:
                raise UsageError("error: unknown option `%s'" % a)
            continue
        # short options, possibly grouped (-dz, -9z, -tbzip2)
        j = 1
        while j < len(a):
            f = a[j]
            j += 1
            if f == "h":
                return {"help": True}
            if f == "V":
                return {"version": True}
            if f == "d":
                opts["decompress"] = True
            elif f == "z":
                opts["compress"] = True
            elif f.isdigit() and f != "0":
                opts["levels"].add(int(f))
            elif f in ("b", "t"):
                val = a[j:]
                if not val:
                    if i >= len(argv):
                        raise UsageError("error: option `%s' argument missing" % ("-b, --block <n>" if f == "b" else "-t <compressor>"))
                    val = argv[i]
                    i += 1
                opts["block" if f == "b" else "T"] = val
                break
            else:
                raise UsageError("error: unknown option `-%s'" % f)
    return opts


def check(opts):
    """bin/compressjs:32-58: returns (decompress, level, block) or raises UsageError with the reference's message."""
    decompress = opts["decompress"]
    compress = opts["compress"] or not decompress
    if decompress and compress:
        raise UsageError("Must specify either -d or -z.")
    block = _number(opts["block"])
    if compress and block >= 0:
        raise UsageError("--block can only be used with decompression")
    level = None
    for l in range(1, 10):
        if l in opts["levels"]:
            if level:
                raise UsageError("Can't specify both -%d and -%d" % (level, l))
            level = l
    if level and decompress:
        raise UsageError("Compression level has no effect when decompressing.")
    return decompress, level or 7, block


def check_recover(opts):
    """--recover / --repair: None without them, else "recover" or "repair"; UsageError when the other options do not
    allow them (they take -d -t bzip2 and nothing else)."""
    rec, rep = opts["recover"], opts["repair"]
    if not (rec or rep):
        return None
    if rec and rep:
        raise UsageError("--recover and --repair cannot be used together")
    flag = "--recover" if rec else "--repair"
    if not opts["decompress"] or opts["compress"]:
        raise UsageError("%s can only be used with -d -t bzip2" % flag)
    if compressor(opts["T"]) != "bzip2":
        raise UsageError("%s can only be used with -d -t bzip2" % flag)
    if _number(opts["block"]) >= 0:
        raise UsageError("%s cannot be used with --block" % flag)
    if opts["levels"]:
        raise UsageError("%s cannot be used with a compression level" % flag)
    if opts["libbz2"]:
        raise UsageError("%s cannot be used with --libbz2" % flag)
    return "repair" if rep else "recover"


def check_libbz2_decode(opts):
    """--libbz2-decode: whether it is given; UsageError when the other options do not allow it (it takes -d -t bzip2
    and nothing else)."""
    if not opts["libbz2-decode"]:
        return False
    if not opts["decompress"] or opts["compress"] or compressor(opts["T"]) != "bzip2":
        raise UsageError("--libbz2-decode can only be used with -d -t bzip2")
    if _number(opts["block"]) >= 0:
        raise UsageError("--libbz2-decode cannot be used with --block")
    if opts["recover"] or opts["repair"]:
        raise UsageError("--libbz2-decode cannot be used with --recover or --repair")
    if opts["libbz2"]:
        raise UsageError("--libbz2-decode cannot be used with --libbz2")
    return True


# the reference's messages of the decode failures a lost block has
REC_MESSAGES = {"DATA_ERROR": "Data error", "OBSOLETE": "Obsolete (pre 0.9.5) bzip format not supported."}


def recover(in_fd, out, repair):
    """--recover / --repair: Bzip2.recover from the descriptor to the binary file `out` through the streams of
    bin/compressjs.  stderr gets "block at bit <p>: <message>" for every candidate that was walked and is not intact, and
    "<k> of <m> blocks intact"; the exit status is 0 when every walked candidate is intact, else 1."""
    from .bzip2 import Bzip2
    src, dst = InStream(in_fd), OutStream(out)
    try:
        _, blocks = Bzip2.recover(src, dst, repair=repair)
    except Exception as e:
        out.flush()
        sys.stderr.write("%s\n" % e)
        return 1
    dst.flush()
    walked = [b for b in blocks if b.status != "INSIDE"]
    intact = sum(b.status == "INTACT" for b in walked)
    for b in walked:
        if b.status == "BAD_CRC":
            sys.stderr.write("block at bit %d: Data error: Bad block CRC (got %x expected %x)\n" % (b.bitpos, b.got, b.crc))
        elif b.status != "INTACT":
            sys.stderr.write("block at bit %d: %s\n" % (b.bitpos, REC_MESSAGES[b.status]))
    sys.stderr.write("%d of %d blocks intact\n" % (intact, len(walked)))
    return 0 if intact == len(walked) else 1


def compressor(name):
    """bin/compressjs:131-158, for the compressors this package has: 'bzip2' or 'bwtc', else UsageError."""
    key = (name if name is not None else "lzp3").lower()
    if key in ("bzip", "bzip2"):
        return "bzip2"
    if key == "bwtc":
        return "bwtc"
    if key in OTHER_COMPRESSORS:
        raise UsageError("Compressor %s is not available in compressjs_b200: use -t bzip2 or -t bwtc" % key)
    raise UsageError("Unknown compressor: %s" % name)


def read_input(fd):
    """(the input's bytes, the size fstat gives): a regular file is mapped, anything else read to its end."""
    st = os.fstat(fd)
    if stat.S_ISREG(st.st_mode) and st.st_size > 0:
        return memoryview(mmap.mmap(fd, 0, access=mmap.ACCESS_READ)), st.st_size
    chunks = []
    while True:
        b = os.read(fd, 1 << 20)
        if not b:
            break
        chunks.append(b)
    return b"".join(chunks), st.st_size


class InStream:
    """makeInStream of bin/compressjs:60-98: the descriptor read a chunk at a time, straight into the caller's buffer.
    Like there, it has a ``size`` only when fstat gives one: a regular, non-empty file.  BWTC writes it into its header,
    and "size unknown" for a stream without one (lib/Util.js:119-124)."""

    def __init__(self, fd):
        self.fd = fd
        st = os.fstat(fd)
        if stat.S_ISREG(st.st_mode) and st.st_size > 0:
            self.size = st.st_size

    def read(self, buf, bufOffset, length):
        """buf: a writable bytes-like object.  Returns the bytes read, 0 at the end of the input."""
        return os.readv(self.fd, [memoryview(buf)[bufOffset:bufOffset + length]]) if length > 0 else 0

    def readByte(self):
        b = os.read(self.fd, 1)
        return b[0] if b else -1


class OutStream:
    """makeOutStream of bin/compressjs:100-116: a FLUSH-byte buffer in front of the binary file `f`, flushed only when
    the next byte arrives (or by flush()).  After T >= 1 bytes, the file has the first FLUSH * ((T - 1) // FLUSH)."""

    def __init__(self, f):
        self.f = f
        self.pending = bytearray()

    def writeByte(self, b):
        if len(self.pending) >= FLUSH:
            self.f.write(self.pending)
            self.pending = bytearray()
        self.pending.append(b & 0xFF)

    def write(self, buf, bufOffset, length):
        """writeByte of each of buf[bufOffset:bufOffset + length], with whole buffers written at once."""
        data = memoryview(bytes(buf) if isinstance(buf, list) else buf).cast("B")[bufOffset:bufOffset + length]
        total = len(self.pending) + len(data)
        cut = total - ((total - 1) % FLUSH + 1) if total else 0   # what goes to the file: whole buffers
        if cut:
            head = cut - len(self.pending)   # >= 0: the pending buffer is at most FLUSH bytes
            self.f.write(self.pending)
            self.f.write(data[:head])
            self.pending = bytearray(data[head:])
        else:
            self.pending += data
        return length

    def flush(self):
        self.f.write(self.pending)
        self.pending = bytearray()
        self.f.flush()


def stream(kind, decompress, level, in_fd, out, flavor="compressjs"):
    """Without -b: compressFile / decompressFile of `kind` ('bzip2' or 'bwtc') from the descriptor to the binary file
    `out` through the streams of bin/compressjs, in bounded memory.  The exit status; on an error its message is on
    stderr and `out` has what went out before it (on a decode error: the decoded bytes cut down to a multiple of FLUSH).
    A bzip2 decode of the libbz2 flavor reads every member, as bzip2 -d does."""
    from .bwtc import BWTC
    from .bzip2 import Bzip2
    src, dst = InStream(in_fd), OutStream(out)
    try:
        if kind == "bwtc":
            if decompress:
                BWTC.decompressFile(src, dst)
            else:
                BWTC.compressFile(src, dst, level)   # the header's size field comes from src.size
        elif decompress and flavor == "libbz2":
            Bzip2.decompressFile(src, dst, True, flavor=flavor)
        elif decompress:
            Bzip2.decompressFile(src, dst)   # without multistream, as bin/compressjs:160-164 calls it
        else:
            Bzip2.compressFile(src, dst, level, flavor=flavor)
    except Exception as e:
        out.flush()
        sys.stderr.write("%s\n" % e)
        return 1
    dst.flush()
    return 0


def run(kind, decompress, level, block, data, size):
    """The whole input at once, as -b needs it: (output bytes, error or None).  On a decode error the bytes are those
    decoded before it."""
    from . import bwtc, bzip2
    from .bwtc import BWTC
    from .bzip2 import Bzip2
    if not decompress:
        if kind == "bzip2":
            return Bzip2.compressFile(data, None, level), None
        if size > 0:
            return BWTC.compressFile(data, None, level), None
        return bwtc._compress_unsized(data, level), None
    if kind == "bzip2":
        # Bzip2.decompressBlock / decompressFile (without multistream, as bin/compressjs:160-164 calls it)
        out, err = bzip2._block(data, int(block)) if block >= 0 else bzip2._file(data)
        return out.tobytes(), err
    if block >= 0:
        raise UsageError("--block needs -t bzip2: compressjs has no BWTC.decompressBlock")
    try:
        return BWTC.decompressFile(data), None
    except (RuntimeError, ValueError) as e:
        return b"", e


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    try:
        opts = parse(argv)
        if opts.get("help"):
            sys.stdout.write(HELP + "\n")
            return 0
        if opts.get("version"):
            sys.stdout.write(VERSION + "\n")
            return 0
        lb_dec = check_libbz2_decode(opts)
        rec = check_recover(opts)
        decompress, level, block = check(opts)
        args = opts["args"]
        in_fd = os.open(args[0], os.O_RDONLY) if len(args) > 0 else sys.stdin.fileno()
        out = open(args[1], "wb") if len(args) > 1 else sys.stdout.buffer
        kind = compressor(opts["T"])
        if opts["libbz2"] and (decompress or kind != "bzip2"):
            raise UsageError("--libbz2 can only be used with -z -t bzip2")
        if rec:
            return recover(in_fd, out, rec == "repair")
        if block < 0:
            return stream(kind, decompress, level, in_fd, out, "libbz2" if opts["libbz2"] or lb_dec else "compressjs")
        data, size = read_input(in_fd)
        result, err = run(kind, decompress, level, block, data, size)
        if err is not None:
            k = len(result)
            out.write(result[:FLUSH * ((k - 1) // FLUSH)] if k else b"")
            out.flush()
            sys.stderr.write("%s\n" % err)
            return 1
        out.write(result)
        out.flush()
        return 0
    except Exception as e:   # usage errors, files that cannot be opened, the library's own errors (no GPU, ...)
        sys.stderr.write("%s\n" % e)
        return 1
