"""LZMA2 options across the branches of the parser kernels and the LZMA2 decoder kernel (-m gpu).

Every sweep case is a multi-Block Stream whose bytes must equal the unmodified reference's lzma_stream_encoder_mt with
the same options (SHA-256 in the opt_sweep section of tests/golden/ref_live_golden.json, recorded by
tests/golden/make_ref_golden.py), and must decode back to its input, alone and all together in one batch.  The
dict_header cases decode Streams whose Block Headers announce other dictionary sizes than the encoder used, and must
give the reference decoder's verdict and the bytes it delivers before it stops.

The inputs are seeded and made here (nothing but hashes is stored):
  ladder       earlier copies that each match one byte longer than the next: match lists of well over 32 pairs, so
               the DP parser walks past its 32-candidate fast path and the match store spills into its overflow pool;
  runs         short-period runs: overlapping copies, rep0 matches of length 273, short reps, and copies of under
               32 and over 32 bytes in the decoder;
  window_edge  300 bytes repeated at exactly `gap`, with gap one below, at and one above the dictionary size.
"""
import functools
import random
import struct
import zlib
from collections import namedtuple

import pytest

import xzlibs as X

pytestmark = [pytest.mark.gpu]
KiB, MiB = 1 << 10, 1 << 20
HC3, HC4, BT2, BT3, BT4 = 0x03, 0x04, 0x12, 0x13, 0x14
FAST, NORMAL = 1, 2
CHECK_SHA256 = 10
CHECKS = (X.CHECK_NONE, X.CHECK_CRC32, X.CHECK_CRC64, CHECK_SHA256)
EDGE_LEN = 300

# name: unique label; blocks: the generator of each Block, in order (the input is their concatenation)
SweepCase = namedtuple("SweepCase", "name opts check block_size blocks data")


# ---- input generators ----

def ladder(n, seed, top=273):
    """For each fresh random base of top + 1 bytes: base[:k] + (base[k] ^ 0xFF) for k from `top` down to 2 in steps
    of 1 to 3, then the whole base.  Seen from the last copy, every earlier copy matches one byte longer than the
    one after it."""
    rnd = random.Random(seed)
    out = bytearray()
    while len(out) < n:
        base = rnd.randbytes(top + 1)
        k = top
        while k >= 2:
            out += base[:k] + bytes([base[k] ^ 0xFF])
            k -= rnd.randint(1, 3)
        out += base
    return bytes(out[:n])


def runs(n, seed):
    """Runs of period 1 to 40, each 1 to 700 bytes long, salted with random bytes."""
    rnd = random.Random(seed)
    out = bytearray()
    while len(out) < n:
        period = rnd.randint(1, 40)
        unit = rnd.randbytes(period)
        length = rnd.randint(1, 700)
        out += (unit * (length // period + 1))[:length]
        if rnd.random() < 0.5:
            out += rnd.randbytes(rnd.randint(1, 3))
    return bytes(out[:n])


def window_edge(gap, n, seed):
    """EDGE_LEN random bytes, random filler, the same EDGE_LEN bytes again at distance exactly `gap`, random filler
    up to n bytes."""
    assert n >= gap + EDGE_LEN and gap >= EDGE_LEN
    rnd = random.Random(seed)
    head = rnd.randbytes(EDGE_LEN)
    return head + rnd.randbytes(gap - EDGE_LEN) + head + rnd.randbytes(n - gap - EDGE_LEN)


def make_block(spec):
    kind, n, arg = spec
    if kind == "ladder":
        return ladder(n, arg)
    if kind == "runs":
        return runs(n, arg)
    if kind == "edge":
        return window_edge(arg[0], n, arg[1])
    return bytes(X.gendata(kind, n, arg)[:n])


# ---- the sweep ----

def opts(mode, mf, nice, depth=0, dict_size=1 * MiB, lc=3, lp=0, pb=2):
    return X.LzmaOptions(dict_size, lc, lp, pb, mode, nice, mf, depth)


def _blocks(i, bs, count=None):
    """2 to 4 Blocks of bs bytes, the last one short, from generators cycling with the case index."""
    count = count or 2 + i % 3
    gens = ["ladder", "runs", "TERL"[i % 4], "runs" if i % 2 else "ladder"]
    specs = []
    for b in range(count):
        n = bs if b < count - 1 else bs // 2 + 1 + 37 * (i % 7)
        kind = gens[b % len(gens)]
        specs.append((kind, n, 1000 * i + b if kind in ("ladder", "runs") else 7919 * i + b * bs))
    return specs


@functools.lru_cache(maxsize=1)
def sweep_cases():
    """The sweep: SweepCase tuples with each case's input built.  The check cycles through None, CRC32, CRC64 and
    SHA-256 in case order."""
    raw = []   # (group, opts, block_size)
    bs = 48 * KiB
    for nice in (2, 3, 4, 5, 7, 8, 9, 16, 31, 32, 33, 63, 64, 126, 127, 128, 129, 191, 192, 255, 256, 272, 273):
        raw.append(("bt4", opts(NORMAL, BT4, nice), bs))
    for mf in (HC3, HC4, BT2, BT3):
        for nice in (2, 3, 8, 32, 127, 128, 273):
            raw.append(("normal", opts(NORMAL, mf, nice), bs))
    for mf in (HC3, HC4, BT2, BT4):
        for nice in (2, 3, 8, 32, 127, 128, 273):
            raw.append(("fast", opts(FAST, mf, nice), bs))
    for mf in (HC4, BT4):
        for mode in (FAST, NORMAL):
            for depth in (1, 2, 3, 200, 5000):
                raw.append(("depth", opts(mode, mf, 128, depth), bs))
    k = 0
    for lc in range(5):
        for lp in range(5 - lc):
            for mode, mf in ((FAST, HC4), (NORMAL, BT4)):
                raw.append(("lclppb", opts(mode, mf, 64, lc=lc, lp=lp, pb=k % 5), bs))
            k += 1
    cases = [(f"{group}-{i}", o, b, _blocks(i, b)) for i, (group, o, b) in enumerate(raw)]
    # the coder-warp form of the fast kernel: a wave with more Blocks than the H100's 132 SMs
    for nice in (2, 273):
        i = len(cases)
        cases.append((f"coderwarp-{i}", opts(FAST, HC4, nice), 2 * KiB, _blocks(i, 2 * KiB, count=150)))
    # window edges: a repeat at dict - 1, dict and dict + 1 in separate Blocks
    for d in (4096, 4097, 6000, 65535, 65537, 1 * MiB - 1):
        for mf in (HC4, BT4):
            i = len(cases)
            full = d + 1 + EDGE_LEN + 16
            blocks = [("edge", full, (d + 1, i)), ("edge", full, (d, i + 1)), ("edge", d - 1 + EDGE_LEN, (d - 1, i + 2))]
            cases.append((f"dict-{i}", opts(NORMAL if mf == BT4 else FAST, mf, 64, dict_size=d), full, blocks))
    # 24-bit hashes, and waves at the 255-Block cap of the (block << 24) sort keys: HC3 keeps 24 bits above 16 MiB,
    # HC4 / BT4 halve the mask at 64 MiB
    for mode, mf, d in ((FAST, HC3, 16 * MiB + 1), (NORMAL, BT4, 64 * MiB)):
        i = len(cases)
        cases.append((f"hash24-{i}", opts(mode, mf, 64, dict_size=d), 4 * KiB, _blocks(i, 4 * KiB, count=300)))
    # one Block past the 2 MiB limit of an uncompressed LZMA2 chunk
    for mode, nice in ((NORMAL, 2), (NORMAL, 273), (FAST, 273)):
        i = len(cases)
        n = 3 * MiB
        cases.append((f"large-{i}", opts(mode, BT4 if mode == NORMAL else HC4, nice, dict_size=8 * MiB), n + 1, [("runs", n, i)]))
    out = []
    for i, (name, o, b, specs) in enumerate(cases):
        data = b"".join(make_block(s) for s in specs)
        out.append(SweepCase(name, o, CHECKS[i % 4], b, specs, data))
    return tuple(out)


def key(case):
    o = case.opts
    return f"{case.name}|{o.mode}.{o.mf:x}.{o.nice_len}.{o.depth}.{o.dict_size}.{o.lc}{o.lp}{o.pb}|{case.check}|{case.block_size}|{len(case.data)}"


# ---- Streams with another dictionary size in their Block Headers ----

DICT_PROPS = tuple(range(41)) + (41, 0xFF)


def dict_header_streams():
    """(name, options, block size, input) of the Streams whose Block Headers are rewritten: single-Block window_edge
    Streams encoded with a dictionary that reaches the repeat, and one multi-Block text Stream."""
    out = []
    for gap in (4095, 4096, 4097, 6144, 6145, 1 * MiB, 1 * MiB + 1):
        n = gap + EDGE_LEN + 100
        out.append((f"edge{gap}", opts(NORMAL, BT4, 64, dict_size=max(gap, 4096)), n, window_edge(gap, n, gap)))
    n = 600 * KiB + 5
    out.append(("T8M", opts(NORMAL, BT4, 64, dict_size=8 * MiB), 256 * KiB, bytes(X.gendata("T", n)[:n])))
    return out


def _index_records(xz):
    back = (struct.unpack_from("<I", xz, len(xz) - 8)[0] + 1) * 4
    count, p = X._read_vli(xz, len(xz) - 12 - back + 1)
    recs = []
    for _ in range(count):
        unpadded, p = X._read_vli(xz, p)
        _, p = X._read_vli(xz, p)
        recs.append(unpadded)
    return recs


def set_dict_prop(xz, prop):
    """The same Stream with the LZMA2 dictionary property byte of every Block Header set to `prop` and the header's
    CRC32 rewritten."""
    out = bytearray(xz)
    check = xz[7] & 0x0F
    pos = 12
    for unpadded in _index_records(xz):
        hs = (out[pos] + 1) * 4
        flags = out[pos + 1]
        assert flags & 0x03 == 0, "one filter: LZMA2"
        q = pos + 2
        if flags & 0x40:
            _, q = X._read_vli(out, q)
        if flags & 0x80:
            _, q = X._read_vli(out, q)
        assert out[q] == 0x21 and out[q + 1] == 1
        out[q + 2] = prop
        struct.pack_into("<I", out, pos + hs - 4, zlib.crc32(bytes(out[pos:pos + hs - 4])))
        pos += (unpadded + 3) & ~3
    assert out[pos] == 0 and check in CHECKS
    return bytes(out)


# ---- GPU tests ----

@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


def _as_product(o):
    import xz_b200
    return xz_b200.LzmaOptions(*[getattr(o, f) for f, _ in X.LzmaOptions._fields_])


_streams = {}


def _encode(ctx, case):
    if case.name not in _streams:
        _streams[case.name] = ctx.stream_encode(case.data, block_size=case.block_size, check=case.check, opts=_as_product(case.opts))
    return _streams[case.name]


@pytest.mark.parametrize("i", range(len(sweep_cases())), ids=[c.name for c in sweep_cases()])
def test_sweep_encode_identical_and_decode(ctx, i):
    case = sweep_cases()[i]
    got = _encode(ctx, case)
    assert X.sha64(got) == X.ref_golden()["opt_sweep"][key(case)], key(case)
    r, back = ctx.stream_decode(got, len(case.data))
    assert r == 0 and back == case.data, key(case)


def test_sweep_batch_decode(ctx):
    """Every sweep Stream in one stream_buffer_decode_batch call: per-job lc/lp/pb, dictionary sizes and checks side
    by side in the same xzb_k_decode launches."""
    cases = sweep_cases()
    gold = X.ref_golden()["opt_sweep"]
    streams = [_encode(ctx, c) for c in cases]
    for c, s in zip(cases, streams):
        assert X.sha64(s) == gold[key(c)], key(c)
    got = ctx.stream_buffer_decode_batch(streams, [len(c.data) for c in cases])
    for c, s, g in zip(cases, streams, got):
        assert g[0] == 0 and g[2] == len(s) and g[1] == c.data, key(c)


def test_dict_header_verdicts(ctx):
    """Block Headers announcing dictionaries from 4 KiB to 4 GiB - 1 (and invalid ones) over Streams that use
    distances up to the encoder's dictionary: the reference decoder's verdict, and the bytes it delivers before a
    match beyond the announced dictionary, from the single decode and from the batch decoder."""
    gold = X.ref_golden()["dict_header"]
    variants, want = [], []
    for name, o, bs, data in dict_header_streams():
        xz = ctx.stream_encode(data, block_size=bs, opts=_as_product(o))
        assert X.sha64(xz) == gold[name]["stream"], name
        for prop in DICT_PROPS:
            v = set_dict_prop(xz, prop)
            ref = gold[name]["props"][str(prop)]
            r, out = ctx.stream_decode(v, len(data))
            assert [r, len(out), X.sha64(out)] == ref, (name, prop)
            variants.append(v); want.append((name, prop, ref, len(data)))
    got = ctx.stream_buffer_decode_batch(variants, [w[3] for w in want])
    for (name, prop, ref, _), g in zip(want, got):
        assert [g[0], len(g[1]), X.sha64(g[1])] == ref, (name, prop)


def test_hash24_batch_equals_single_calls(ctx):
    """300 one-shot Streams with 24-bit hashes: two waves under the 255-Block cap of the (block << 24) sort keys give
    the bytes of 300 single calls."""
    case = [c for c in sweep_cases() if c.name.startswith("hash24") and c.opts.mf == HC3][0]
    o = _as_product(case.opts)
    items, p = [], 0
    for kind, n, _ in case.blocks:
        items.append(case.data[p:p + n]); p += n
    assert len(items) == 300
    got = ctx.stream_buffer_encode_batch(items, check=case.check, opts=o)
    for k, it in enumerate(items):
        assert got[k] == (0, ctx.stream_buffer_encode(it, check=case.check, opts=o)), k
