#!/usr/bin/env python
"""Batch one-shot encode / decode against a loop of single calls, on SquashFS-like jobs.

Jobs: 4096 x 128 KiB of `T` at -6 with CRC32 (one Stream per filesystem block), and 1024 x 1 MiB of `T` at -1 with
CRC64.  For each job the probe reports MB/s of uncompressed data for
  * the batch: device-timed (CUDA events of the call, xzb_stats.ms_total) and end to end (host clock around the
    Python call, packing of the items and copies included);
  * a loop of single calls (xzb_stream_buffer_encode / _decode) over the first `--loop` items only, end to end;
  * device-resident decode (xzb_stream_buffer_decode_batch_device) of the Streams that the device encode batch left in
    HBM, into slots in HBM: device-timed, and end to end (host clock around the call, which ends in a synchronise).
Every batch item is checked against the single call on that subset, and both batch decodes against the input.
The card's name and power limit are read in the same run.  Prints one JSON line; --out DIR also writes it there.

    python profiles/batch_probe.py [--loop 64] [--out DIR]
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

KiB, MiB = 1 << 10, 1 << 20
JOBS = (("squashfs_128k_-6_crc32", 4096, 128 * KiB, 6, 1), ("1m_-1_crc64", 1024, MiB, 1, 4))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_job(ctx, name, count, size, preset, check, loop):
    import xzlibs as X
    whole = bytes(X.gendata("T", count * size)[:count * size])
    items = [whole[i * size:(i + 1) * size] for i in range(count)]
    total = count * size
    sub = items[:loop]
    ctx.stream_buffer_encode_batch(sub[:8], preset=preset, check=check)  # warm-up: modules, workspace
    t0 = time.perf_counter()
    enc = ctx.stream_buffer_encode_batch(items, preset=preset, check=check)
    t_enc = time.perf_counter() - t0
    enc_dev_ms = ctx.stats().ms_total
    assert all(r == 0 for r, _ in enc)
    streams = [xz for _, xz in enc]
    t0 = time.perf_counter()
    single = [ctx.stream_buffer_encode(x, preset=preset, check=check) for x in sub]
    t_enc_loop = time.perf_counter() - t0
    assert single == streams[:loop], "batch and single calls differ"
    caps = [size] * count
    ctx.stream_buffer_decode_batch(streams[:8], caps[:8])
    t0 = time.perf_counter()
    dec = ctx.stream_buffer_decode_batch(streams, caps)
    t_dec = time.perf_counter() - t0
    dec_dev_ms = ctx.stats().ms_total
    assert [(r, out) for r, out, _ in dec] == [(0, x) for x in items], "batch decode did not return the items"
    t0 = time.perf_counter()
    for s in streams[:loop]:
        r, out, _ = ctx.stream_buffer_decode(s, size)
        assert r == 0
    t_dec_loop = time.perf_counter() - t0
    dd_dev_ms, t_dd = device_decode(ctx, whole, count, size, preset, check)
    mbs = lambda nbytes, sec: round(nbytes / sec / 1e6, 2)
    return {"job": name, "items": count, "item_bytes": size, "preset": preset, "check": check,
            "ratio": round(total / sum(len(s) for s in streams), 3),
            "encode_batch_MBps_device": mbs(total, enc_dev_ms / 1e3), "encode_batch_MBps_e2e": mbs(total, t_enc),
            "encode_loop_MBps_e2e": mbs(loop * size, t_enc_loop),
            "decode_batch_MBps_device": mbs(total, dec_dev_ms / 1e3), "decode_batch_MBps_e2e": mbs(total, t_dec),
            "decode_loop_MBps_e2e": mbs(loop * size, t_dec_loop), "loop_items": loop,
            "decode_device_batch_MBps_device": mbs(total, dd_dev_ms / 1e3), "decode_device_batch_MBps_e2e": mbs(total, t_dd)}


def device_decode(ctx, whole, count, size, preset, check):
    """(device ms, host seconds) of the device-resident decode of the job's Streams, made by the device encode batch."""
    import xz_b200
    cap = xz_b200.lib().xzb_stream_buffer_bound(size)
    d_src, d_xz, d_back = ctx.device_alloc(len(whole)), ctx.device_alloc(cap * count), ctx.device_alloc(len(whole))
    try:
        ctx.h2d(d_src, whole, len(whole))
        offs = [i * size for i in range(count)]
        xz_offs = [i * cap for i in range(count)]
        enc = ctx.stream_buffer_encode_batch_device(d_src, offs, [size] * count, xz_b200.lzma_lzma_preset(preset), check, d_xz, xz_offs,
                                                    [cap] * count)
        assert all(r == 0 for r, _ in enc)
        sizes = [s for _, s in enc]
        ctx.stream_buffer_decode_batch_device(d_xz, xz_offs[:8], sizes[:8], d_back, offs[:8], [size] * 8)  # warm-up
        t0 = time.perf_counter()
        dec = ctx.stream_buffer_decode_batch_device(d_xz, xz_offs, sizes, d_back, offs, [size] * count)
        t = time.perf_counter() - t0
        dev_ms = ctx.stats().ms_total
        assert dec == [(0, size, s) for s in sizes]
        back = bytearray(len(whole))
        ctx.d2h(back, d_back, len(whole))
        assert bytes(back) == whole, "device decode did not return the items"
    finally:
        ctx.device_free(d_src); ctx.device_free(d_xz); ctx.device_free(d_back)
    return dev_ms, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loop", type=int, default=64, help="items timed as a loop of single calls")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import xz_b200
    ctx = xz_b200.Context(0)
    res = {"card": card(), "jobs": [run_job(ctx, *j, loop=a.loop) for j in JOBS]}
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "batch_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
