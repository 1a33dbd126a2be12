#!/usr/bin/env python
"""Whole-Stream batch encode (xzb_stream_encode_batch) against a loop of single xzb_stream_encode calls.

Jobs:
  (a) 64 x 40 MiB of `T` at -6 with the default Block size (24 MiB): a single call codes an item's two Blocks side by
      side, the batch all 128 Blocks in shared waves;
  (b) 512 x 4 MiB of `E` at -1 in 1 MiB Blocks: the batch, a loop of single calls, and the one-shot batch
      (xzb_stream_buffer_encode_batch: one 4 MiB Block per item) of the same items.
For each it reports MB/s of uncompressed data, device-timed (CUDA events of the call, xzb_stats.ms_total) and end to
end (host clock around the Python call, packing of the items and copies included).  The loop runs over the first
`--loop-a` / `--loop-b` items only; the batch's Streams of those items are checked equal to the loop's.  The card's
name, power limit and SM clock are read in the same run.  Prints one JSON line; --out DIR also writes it there.

    python profiles/stream_batch_probe.py [--loop-a 1] [--loop-b 32] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

MiB = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def mbs(nbytes, sec):
    return round(nbytes / sec / 1e6, 3)


def items_of(kind, count, size):
    import xzlibs as X
    whole = bytes(X.gendata(kind, count * size)[:count * size])
    return [whole[i * size:(i + 1) * size] for i in range(count)]


def timed(ctx, fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0, ctx.stats().ms_total / 1e3


def run_job(ctx, name, kind, count, size, preset, block_size, loop, oneshot):
    items = items_of(kind, count, size)
    total, sub = count * size, items[:loop]
    ctx.stream_encode_batch(items[:2], preset=preset, block_size=block_size)   # warm-up: modules, workspace
    batch, t_e2e, t_dev = timed(ctx, lambda: ctx.stream_encode_batch(items, preset=preset, block_size=block_size))
    assert all(r == 0 for r, _ in batch)
    streams = [xz for _, xz in batch]
    t0, dev = time.perf_counter(), 0.0
    single = []
    for x in sub:
        single.append(ctx.stream_encode(x, preset=preset, block_size=block_size))
        dev += ctx.stats().ms_total / 1e3
    t_loop = time.perf_counter() - t0
    assert single == streams[:loop], "batch and single calls differ"
    res = {"job": name, "items": count, "item_bytes": size, "preset": preset, "block_size": block_size or "default",
           "ratio": round(total / sum(len(s) for s in streams), 3),
           "batch_MBps_device": mbs(total, t_dev), "batch_MBps_e2e": mbs(total, t_e2e),
           "loop_items": loop, "loop_MBps_device": mbs(loop * size, dev), "loop_MBps_e2e": mbs(loop * size, t_loop)}
    if oneshot:
        one, t_e2e, t_dev = timed(ctx, lambda: ctx.stream_buffer_encode_batch(items, preset=preset))
        assert all(r == 0 for r, _ in one)
        res.update({"oneshot_batch_MBps_device": mbs(total, t_dev), "oneshot_batch_MBps_e2e": mbs(total, t_e2e),
                    "oneshot_ratio": round(total / sum(len(s) for _, s in one), 3)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loop-a", type=int, default=1, help="items of job (a) timed as a loop of single calls")
    ap.add_argument("--loop-b", type=int, default=32, help="items of job (b) timed as a loop of single calls")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import xz_b200
    ctx = xz_b200.Context(0)
    res = {"card": card(), "jobs": [run_job(ctx, "a_64x40MiB_T_-6_default", "T", 64, 40 * MiB, 6, 0, a.loop_a, False),
                                    run_job(ctx, "b_512x4MiB_E_-1_1MiB", "E", 512, 4 * MiB, 1, MiB, a.loop_b, True)]}
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "stream_batch_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
