"""Measure the resumable Block decoder (xzb_block_decoder_*) against the whole-Block kernel on the same data.

For each input -- `T` and `E` text (tests/xzlibs.gendata) at -1, and the high-ratio synthetic Block of
tests/test_gpu_block_decoder.py -- one large Block is decoded piece by piece (unsized, output taken in 64 MiB buffers)
and the same bytes as a Stream of sized 4 MiB Blocks at -1 go through xzb_stream_buffer_decode (whole-Block jobs).  The
one large Block is those 4 MiB Blocks' LZMA2 data joined, end markers dropped but the last: this is one valid LZMA2
stream only because every Block's data starts with a dictionary reset (0x01 or 0xE0), as every LZMA2 encoder writes it.
Reported per input: device-timed decode MB/s (the decode kernels' CUDA-event time) and end-to-end MB/s (host clock
around the whole call), and for the piece-by-piece path the per-piece overheads: pieces, model bytes moved (2 x 28 KB
per piece), window slides and bytes slid, check-kernel and output-copy time.  Prints one JSON line per input, with the
card's name and power limit.

    python profiles/block_decoder_probe.py [--mb 64] [--reps 640]     (DESIGN §8 figures: --mb 32 --reps 256)
"""
import argparse
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                              text=True).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def pieces_path(ctx, blk, check, total):
    from test_block_decoder_cpu import header_size
    hs = header_size(blk)
    cap = 64 << 20
    obuf = (C.c_uint8 * cap)()
    src = (C.c_uint8 * len(blk)).from_buffer_copy(blk)
    t0 = time.perf_counter()
    bd = ctx.block_decoder(blk[:hs], check)
    pos, got = hs, 0
    while True:
        r, n, used = bd.code_into(C.addressof(src) + pos, len(blk) - pos, obuf, cap, True)
        pos += used; got += n
        if r != 0:
            break
    t1 = time.perf_counter()
    st = bd.stats().as_dict()
    bd.close()
    assert r == 1 and got == total, (r, got, total)
    return t1 - t0, st


def whole_path(ctx, xz, total):
    out = (C.c_uint8 * (total + 1))()
    import xz_b200
    lib = xz_b200.lib()
    sz, used = C.c_uint64(), C.c_uint64()
    src = (C.c_uint8 * len(xz)).from_buffer_copy(xz)
    t0 = time.perf_counter()
    r = lib.xzb_stream_buffer_decode(ctx._h, src, len(xz), out, total + 1, C.byref(sz), C.byref(used), 0)
    t1 = time.perf_counter()
    assert r == 0 and sz.value == total
    return t1 - t0, ctx.stats().ms_decode


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=64, help="MiB of T / E text")
    ap.add_argument("--reps", type=int, default=640, help="0xA0 chunks of the synthetic Block (2 MiB of output each)")
    a = ap.parse_args()
    import xz_b200
    import xzlibs as X
    import test_gpu_block_decoder as TB
    ctx = xz_b200.Context(0)
    gpu = card()
    inputs = []
    from test_block_decoder_cpu import blocks, header_size
    for kind in ("T", "E"):
        n = a.mb << 20
        buf = X.gendata(kind, n)
        sized = ctx.stream_encode(buf, preset=1, block_size=4 << 20, check=X.CHECK_CRC32, n=n)
        # one unsized Block holding the same chunks: every Block's LZMA2 data starts with a dictionary reset, so the
        # payloads joined (end markers dropped but the last) are one valid LZMA2 stream of all n bytes
        pl = bytearray()
        for blk, _ in blocks(sized):
            hs = header_size(blk)
            comp, _ = X._read_vli(blk, 2)
            pl += blk[hs: hs + comp - 1]
        pl.append(0)
        one = TB.block_bytes(bytes(pl), n, 1, struct.pack("<I", zlib.crc32(bytes(buf[:n]))), False)
        inputs.append((kind, one, sized, n))
    payload, headb, fill, total = TB.synthetic(a.reps)
    cf = TB.expected_check(headb, fill, total, 1)
    blk = TB.block_bytes(payload, total, 1, cf, False)
    inputs.append(("synthetic", blk, None, total))
    for name, blk, sized, total in inputs:
        check = 1
        pieces_path(ctx, blk, check, total)   # warm-up
        e2e, st = pieces_path(ctx, blk, check, total)
        row = {"input": name, "bytes": total, "card": gpu,
               "pieces_e2e_MBps": total / e2e / 1e6, "pieces_device_MBps": total / (st["ms_decode"] / 1e3) / 1e6,
               "pieces": st["pieces"], "model_bytes_moved": st["pieces"] * 2 * 28 * 1024, "slides": st["slides"],
               "bytes_slid": st["bytes_slid"], "window_bytes": st["window_bytes"], "ms_decode": st["ms_decode"],
               "ms_check": st["ms_check"], "ms_d2h": st["ms_d2h"], "e2e_s": e2e}
        if sized is not None:
            whole_path(ctx, sized, total)
            w_e2e, w_ms = whole_path(ctx, sized, total)
            nb = len(blocks(sized))
            # the Blocks run side by side: one Block's rate is its share of the bytes over the launch's time
            row.update({"whole_e2e_MBps": total / w_e2e / 1e6, "whole_device_MBps": total / (w_ms / 1e3) / 1e6,
                        "whole_blocks": nb, "whole_per_block_device_MBps": total / nb / (w_ms / 1e3) / 1e6})
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
