"""Development probe (not a pytest file): normal-mode parser kernel vs the oracle on a handful of inputs,
with a symbol-trace diff on the first mismatch, and the parser's timing on a few multi-Block streams.

    python tests/gpu_probe_dp.py [quick|time|all]
"""
import ctypes as C
import os
import struct
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import xz_b200
if os.environ.get("XZB200_LIB"):
    xz_b200.LIB_PATH = os.path.abspath(os.environ["XZB200_LIB"])   # A/B: a library built with other switches
else:
    import __graft_entry__ as ge
    ge.build()
import xzlibs as X

MiB = 1 << 20
EXT = 0x80000000


def oracle_trace(buf, n, opts):
    lib = X.oracle()
    cap = n + 16
    tr = (C.c_uint32 * (3 * cap))()
    cnt = C.c_size_t()
    lib.xzo_set_trace(tr, C.c_size_t(cap), C.byref(cnt))
    out = X.oracle_encode(buf, n, 0, max(n, 1), opts=opts)
    lib.xzo_set_trace(None, C.c_size_t(0), None)
    return out, [(tr[3 * i], tr[3 * i + 1], tr[3 * i + 2]) for i in range(cnt.value)]


def check(kind, preset, n, bs, opts=None, label=""):
    buf = X.gendata(kind, n)
    o = opts if opts is not None else xz_b200.lzma_lzma_preset(preset)
    oo = X.LzmaOptions()
    for f, _ in X.LzmaOptions._fields_:
        setattr(oo, f, getattr(o, f))
    want = X.oracle_encode(buf, n, preset, bs, opts=oo)
    os.environ.pop("XZB_TRACE", None)
    ctx = xz_b200.Context(0)
    t = time.time()
    got = ctx.stream_encode(buf, preset=preset, block_size=bs, n=n, opts=o)
    dt = time.time() - t
    s = ctx.stats().as_dict()
    ctx.close()
    ok = got == want
    print(f"{'OK ' if ok else 'BAD'} {kind} preset={preset & 31}{'e' if preset & EXT else ''} n={n} bs={bs} {label} "
          f"parse_ms={s['ms_parse']:.1f} total_ms={s['ms_total']:.1f} wall={dt:.2f}s", flush=True)
    if not ok:
        # trace diff on the first block
        n0 = min(n, bs)
        os.environ["XZB_TRACE"] = "/tmp/xzb_trace.bin"
        ctx = xz_b200.Context(0)
        try:
            ctx.stream_encode(buf, preset=preset, block_size=n0, n=n0, opts=o)
        except Exception as ex:
            print("   traced run failed:", ex)
        ctx.close()
        os.environ.pop("XZB_TRACE", None)
        raw = open("/tmp/xzb_trace.bin", "rb").read() if os.path.exists("/tmp/xzb_trace.bin") else b""
        mine = [struct.unpack_from("<III", raw, 12 * i) for i in range(len(raw) // 12)]
        _, ref = oracle_trace(buf, n0, oo)
        k = 0
        while k < min(len(mine), len(ref)) and mine[k] == ref[k]:
            k += 1
        print(f"   first block: {len(mine)} symbols here, {len(ref)} in the oracle; first difference at symbol {k}")
        for j in range(max(0, k - 3), min(max(len(mine), len(ref)), k + 4)):
            a = mine[j] if j < len(mine) else None
            b = ref[j] if j < len(ref) else None
            print(f"   {j}: gpu={a} oracle={b}")
    return ok


def quick():
    ok = True
    ok &= check("T", 6, 300000, 1 << 18)
    ok &= check("E", 6, 1 << 20, 1 << 20)
    ok &= check("R", 6, 200000, 1 << 17)
    ok &= check("T", 4, 1 << 20, 1 << 19)
    ok &= check("E", 9 | EXT, 1 << 21, 1 << 21)
    ok &= check("T", 6, 4 * MiB, 4 * MiB)
    ok &= check("T", 9 | EXT, 1 << 20, 1 << 20)
    ok &= check("L", 6, 1 << 18, 1 << 18)
    for lc, lp, pb in ((0, 2, 0), (4, 0, 4), (1, 3, 1)):
        o = xz_b200.lzma_lzma_preset(6)
        o.lc, o.lp, o.pb = lc, lp, pb
        ok &= check("E", 6, 400000, 1 << 18, opts=o, label=f"lc{lc}lp{lp}pb{pb}")
    for mf in (0x12, 0x13, 0x03, 0x04):
        o = xz_b200.lzma_lzma_preset(6)
        o.mf, o.nice_len, o.depth = mf, 32, 0
        ok &= check("T", 6, 500000, 1 << 18, opts=o, label=f"mf{mf:#x}")
    print("ALL OK" if ok else "FAILURES", flush=True)
    return ok


def timing():
    for kind, preset, nb, bs in (("T", 6, 8, 4 * MiB), ("E", 6, 8, 4 * MiB), ("E", 9 | EXT, 8, 2 * MiB)):
        n = nb * bs
        buf = X.gendata(kind, n)
        ctx = xz_b200.Context(0)
        o = xz_b200.lzma_lzma_preset(preset)
        ctx.stream_encode(buf, preset=preset, block_size=bs, n=n, opts=o)
        ctx.stream_encode(buf, preset=preset, block_size=bs, n=n, opts=o)
        s = ctx.stats().as_dict()
        print(f"time {kind} -{preset & 31} {nb}x{bs // MiB}MiB: parse_ms={s['ms_parse']:.1f} mf_ms={s['ms_mf']:.1f} total_ms={s['ms_total']:.1f}", flush=True)
        ctx.close()


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    ok = True
    if what in ("quick", "all"):
        ok = quick()
    if what in ("time", "all"):
        timing()
    sys.exit(0 if ok else 1)
