"""The multi-GPU share decode (sharded.decompress_shares' stages) in both decoder flavors.

Eight ranks are simulated on one GPU, as tools/share_dec_run.py and the GPU tests do: every rank's session is opened
and exported, the rows are concatenated, then every rank's session is opened again and finished.  A round's time is the
sum over the ranks of the first open (scan, decode and export) and of the finish (walk, expand and CRC check), each the
host wall clock of one call that ends in a device synchronise; the slowest rank's open and finish are printed too.
Every round's output is placed at the ranks' offsets and compared with the expected bytes.

  (a) the config-2 stream (tests/util.py ascii_random, as bench.py's config 2), compressed at level 9 on the GPU:
      one warm-up round per flavor, then the two flavors alternated, three rounds each; medians.
  (b) about 256 MiB of decoded output in members of one randomised 900 000-byte block each (the file of
      tests/test_gpu_libbz2_decode.py's scale test), libbz2 flavor only: one warm-up round, three rounds; median.

The card's name and power limit, read in the same run, head the output.

    python tools/libbz2_share_dec_run.py [GiB] [ranks]      (default 1 GiB, 8 simulated ranks)
"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from share_dec_run import card, placed, stream, timed  # noqa: E402


def shares_round(host, exp_dev, world, flavor, multistream):
    """One share decode of `host` (pinned uint8 tensor) by `world` simulated ranks: dict of times and the check."""
    from compressjs_b200 import sharded as S
    n = host.numel()
    g0s = [r * n // world for r in range(world)]
    lens = [(r + 1) * n // world - g0s[r] for r in range(world)]
    holds = [min(n - g0, ln + S.DEC_HALO) for g0, ln in zip(g0s, lens)]
    bufs = [host[g0: g0 + h].cuda() for g0, h in zip(g0s, holds)]
    rows, t_open = [], []
    for r in range(world):
        (rw, rc, msg), ms = timed(lambda: S._share_open(bufs[r], lens[r], g0s[r], n, flavor))
        assert rc == 0, msg
        rows.append(rw)
        t_open.append(ms)
    all_rows = torch.cat(rows)
    pieces, t_fin = [], []
    for r in range(world):
        S._share_open(bufs[r], lens[r], g0s[r], n, flavor)
        (o, info), ms = timed(lambda: S._share_finish(all_rows, rows[r], multistream, bufs[r].device, flavor))
        assert o is not None and not info["unsettled"], info
        pieces.append((info["off"], o))
        t_fin.append(ms)
    return dict(ms=sum(t_open) + sum(t_fin), open_ms=sum(t_open), finish_ms=sum(t_fin), slowest_open_ms=max(t_open),
                slowest_finish_ms=max(t_fin), identical=placed(pieces, exp_dev))


def summary(rounds):
    keys = ("ms", "open_ms", "finish_ms", "slowest_open_ms", "slowest_finish_ms")
    return dict({k: statistics.median(r[k] for r in rounds) for k in keys}, all_ms=[round(r["ms"], 1) for r in rounds],
                identical=all(r["identical"] for r in rounds))


def randomised_members():
    from tests import bz2synth as W
    from tests import libbz2_read_cases as LC
    from tests import util as T
    members, outs = [], []
    for s in range(3):
        P = np.frombuffer(T.ascii_random(900000, 500 + s), np.uint8)
        members.append(W.Member([LC.rand_block(P)], 9).data)
        outs.append(W.model_rle1(P)[0].tobytes())
    k = (256 << 20) // 900000
    return b"".join(outs[i % 3] for i in range(k)), b"".join(members[i % 3] for i in range(k))


def main():
    gib = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    world = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    if not torch.cuda.is_available():
        raise SystemExit("libbz2_share_dec_run: no CUDA device")
    for line in card():
        print("card:", line)
    out = {"simulated_ranks": world}
    data, z = stream(gib)
    print("(a) config-2 bytes: %d, level-9 stream: %d bytes" % (len(data), len(z)))
    host = torch.frombuffer(bytearray(z), dtype=torch.uint8).pin_memory()
    exp_dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    del data
    flavors = ("compressjs", "libbz2")
    for fl in flavors:
        shares_round(host, exp_dev, world, fl, False)   # warm-up
    rounds = {fl: [] for fl in flavors}
    for _ in range(3):
        for fl in flavors:
            rounds[fl].append(shares_round(host, exp_dev, world, fl, False))
    for fl in flavors:
        out["config2_" + fl] = s = summary(rounds[fl])
        print("  %-10s median %.1f ms (rounds %s), open %.1f ms, finish %.1f ms, slowest rank open %.1f ms, finish %.1f ms, "
              "identical: %s" % (fl, s["ms"], s["all_ms"], s["open_ms"], s["finish_ms"], s["slowest_open_ms"], s["slowest_finish_ms"],
                                 s["identical"]))
    del host, exp_dev
    data, z = randomised_members()
    print("(b) randomised members: %d decoded bytes, %d compressed bytes" % (len(data), len(z)))
    host = torch.frombuffer(bytearray(z), dtype=torch.uint8).pin_memory()
    exp_dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    shares_round(host, exp_dev, world, "libbz2", True)   # warm-up
    out["randomised_members_libbz2"] = s = summary([shares_round(host, exp_dev, world, "libbz2", True) for _ in range(3)])
    print("  libbz2     median %.1f ms (rounds %s), %.2f GB/s of decoded output, open %.1f ms, finish %.1f ms, identical: %s"
          % (s["ms"], s["all_ms"], len(data) / s["ms"] / 1e6, s["open_ms"], s["finish_ms"], s["identical"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
