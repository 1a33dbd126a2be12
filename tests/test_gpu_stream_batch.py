"""GPU tests (-m gpu) of the whole-Stream batch (xzb_stream_encode_batch[_device]): every item of a batch gets the
lzma_stream_encoder_mt Stream that xzb_stream_encode gives it alone -- the reference's bytes for the recorded Streams
(tests/golden/encode_golden.json, and the chain_encode and chunk_mix sections of tests/golden/ref_live_golden.json),
the single call's bytes for seeded batches of mixed sizes whose Blocks share waves or span many -- from host and from
device memory, with a slot one byte short failing alone, and every Stream decodes back to its input."""
import hashlib
import json
import os
import random

import pytest

import chunk_mix as M
import xzlibs as X
from test_gpu_filters import chain_cases

pytestmark = pytest.mark.gpu
GOLD = os.path.join(X.ROOT, "tests", "golden")
OK, UNSUPPORTED_CHECK, OPTIONS_ERROR, BUF_ERROR = 0, 3, 8, 10
KiB, MiB = 1 << 10, 1 << 20


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


def _data(kind, n):
    return bytes(X.gendata(kind, n)[:n])


def _product_opts(o):
    import xz_b200
    return xz_b200.LzmaOptions(*[getattr(o, f) for f, _ in X.LzmaOptions._fields_])


def _decode_all(ctx, streams, items):
    """Every Stream through xzb_stream_buffer_decode_batch_device gives its input back."""
    n = len(streams)
    in_off, out_off, at, out_at = [], [], 0, 0
    for s, x in zip(streams, items):
        in_off.append(at); at += len(s)
        out_off.append(out_at); out_at += len(x) + 1
    d_in, d_out = ctx.device_alloc(max(at, 1)), ctx.device_alloc(max(out_at, 1))
    try:
        blob = b"".join(streams)
        if blob:
            ctx.h2d(d_in, blob, len(blob))
        got = ctx.stream_buffer_decode_batch_device(d_in, in_off, [len(s) for s in streams], d_out, out_off, [len(x) + 1 for x in items])
        back = bytearray(max(out_at, 1))
        ctx.d2h(back, d_out, max(out_at, 1))
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    for i in range(n):
        assert got[i][0] == OK and got[i][1] == len(items[i]) and got[i][2] == len(streams[i]), i
        assert bytes(back[out_off[i]: out_off[i] + len(items[i])]) == items[i], i


def test_batches_match_reference_golden(ctx):
    """The 249 recorded lzma_stream_encoder_mt Streams, one batch per (preset, block size, check), shuffled, with one
    item twice: sizes 0 to 16 MiB + 1, block sizes 256 KiB to 16 MiB, -0 to -9e."""
    cases = json.load(open(os.path.join(GOLD, "encode_golden.json")))
    groups = {}
    for c in cases:
        groups.setdefault((c["preset"], c["block_size"], c["check"]), []).append(c)
    assert sum(len(g) for g in groups.values()) == 249
    rng = random.Random(23)
    for (preset, bs, check), g in sorted(groups.items()):
        g = g + [g[len(g) // 2]]
        rng.shuffle(g)
        out = ctx.stream_encode_batch([_data(c["kind"], c["size"]) for c in g], preset=preset, block_size=bs, check=check)
        for c, (r, xz) in zip(g, out):
            assert r == OK and len(xz) == c["xz_size"] and hashlib.sha256(xz).hexdigest() == c["xz_sha256"], (preset, bs, c["kind"], c["size"])


def test_filter_chain_batches_match_reference(ctx):
    """The chain_encode Streams, each input twice in one batch beside an empty item, with the chain on the context."""
    for chain, preset, n, bs, data in chain_cases():
        ctx.set_filters(chain)
        try:
            out = ctx.stream_encode_batch([data, b"", data], preset=preset, block_size=bs)
        finally:
            ctx.set_filters(())
        want = X.ref_golden()["chain_encode"]["+".join(f"{i:x}.{a:x}" for i, a in chain) + f"|{preset}|{n}|{bs}"]
        assert [r for r, _ in out] == [OK] * 3
        assert X.sha64(out[0][1]) == want and out[2][1] == out[0][1], chain
        assert out[1][1] == X.oracle_encode(X.gendata("T", 0), 0, preset, bs)


def test_chunk_mix_batches_match_reference(ctx):
    """The chunk_mix cases batched per (options, check, block size), each case's input twice: incompressible Blocks
    and Blocks that switch between LZMA and uncompressed chunks, 288 Blocks in one wave for the coder-warp form."""
    groups = {}
    for case in M.cases():
        o = case.opts
        groups.setdefault((tuple(getattr(o, f) for f, _ in X.LzmaOptions._fields_), case.check, case.block_size), []).append(case)
    for (_, check, bs), g in groups.items():
        g = g + g
        out = ctx.stream_encode_batch([c.data for c in g], block_size=bs, check=check, opts=_product_opts(g[0].opts))
        for c, (r, xz) in zip(g, out):
            assert r == OK and X.sha64(xz) == X.ref_golden()["chunk_mix"][M.key(c)]["stream"], M.key(c)


def _seeded_items(seed, count=150, top=12 * MiB):
    """Sizes 0 .. 12 MiB, log-uniform, 0, 1, 1 MiB, 2 MiB and 12 MiB included; T / E / R data."""
    rng = random.Random(seed)
    sizes = [0, 1, MiB, 2 * MiB, top] + [int(top ** rng.random()) for _ in range(count - 5)]
    rng.shuffle(sizes)
    return [_data("TER"[i % 3], s) for i, s in enumerate(sizes)]


@pytest.mark.parametrize("preset", [1, 6])
def test_seeded_batch_equals_single_calls_in_shared_waves_and_many(ctx, monkeypatch, preset):
    """~150 items in 1 MiB Blocks: the batch equals stream_encode of each item alone, with every Block counted once;
    XZB_MAX_WAVE_BLOCKS=7 spreads the same Blocks, an item's Blocks across waves, over many waves."""
    import xz_b200
    items = _seeded_items(preset)
    want = [ctx.stream_encode(x, preset=preset, block_size=MiB) for x in items]
    got = ctx.stream_encode_batch(items, preset=preset, block_size=MiB)
    assert [r for r, _ in got] == [OK] * len(items)
    assert [xz for _, xz in got] == want
    assert ctx.stats().n_blocks == sum((len(x) + MiB - 1) // MiB for x in items)
    monkeypatch.setenv("XZB_MAX_WAVE_BLOCKS", "7")
    c7 = xz_b200.Context(0)
    try:
        got7 = c7.stream_encode_batch(items, preset=preset, block_size=MiB)
        assert [r for r, _ in got7] == [OK] * len(items) and [xz for _, xz in got7] == want
    finally:
        c7.close()
    _decode_all(ctx, want, items)


def test_device_batch_odd_offsets_short_slot_and_canary(ctx):
    """Inputs and slots at odd offsets in device memory pre-filled with a canary; item 3's slot is one byte short: it
    alone gets XZB_BUF_ERROR with size 0, and no byte outside the slots changes.  SHA-256 check, 512 KiB Blocks."""
    import xz_b200
    opts = xz_b200.lzma_lzma_preset(1)
    bs, check = 512 * KiB, 10
    sizes = [3 * MiB + 7, 0, 1, 2 * MiB + 12345, 511 * KiB, 5 * bs, 777777]
    items = [_data("TER"[i % 3], s) for i, s in enumerate(sizes)]
    want = [ctx.stream_encode(x, opts=opts, block_size=bs, check=check) for x in items]
    caps = [xz_b200.stream_bound(len(x), bs) for x in items]
    caps[3] = len(want[3]) - 1
    in_off, at = [], 3
    for x in items:
        in_off.append(at); at += len(x) + 5
    out_off, o = [], 1
    for c in caps:
        out_off.append(o); o += c + 3
    d_in, d_out = ctx.device_alloc(at), ctx.device_alloc(o)
    canary = bytes((0x5A + 7 * k) & 0xFF for k in range(o))
    try:
        blob = bytearray(at)
        for x, p in zip(items, in_off):
            blob[p: p + len(x)] = x
        ctx.h2d(d_in, bytes(blob), at)
        ctx.h2d(d_out, canary, o)
        got = ctx.stream_encode_batch_device(d_in, in_off, sizes, opts, check, bs, d_out, out_off, caps)
        back = bytearray(o)
        ctx.d2h(back, d_out, o)
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    for i, (r, size) in enumerate(got):
        if i == 3:
            assert (r, size) == (BUF_ERROR, 0)
        else:
            assert (r, size) == (OK, len(want[i])) and bytes(back[out_off[i]: out_off[i] + size]) == want[i], i
    inside = bytearray(o)
    for p, c in zip(out_off, caps):
        inside[p: p + c] = b"\1" * c
    assert all(back[k] == canary[k] for k in range(o) if not inside[k])
    ok = [i for i in range(len(items)) if i != 3]
    _decode_all(ctx, [want[i] for i in ok], [items[i] for i in ok])


def test_device_batch_default_block_size_and_no_items(ctx):
    import xz_b200
    opts = xz_b200.lzma_lzma_preset(0)   # 256 KiB dictionary: the default Block is 1 MiB
    items = [_data("T", 2 * MiB + 99), _data("E", 700000)]
    want = [ctx.stream_encode(x, opts=opts, block_size=0) for x in items]
    caps = [xz_b200.stream_bound(len(x), MiB) for x in items]
    d_in, d_out = ctx.device_alloc(sum(len(x) for x in items)), ctx.device_alloc(sum(caps))
    try:
        ctx.h2d(d_in, items[0] + items[1], len(items[0]) + len(items[1]))
        got = ctx.stream_encode_batch_device(d_in, [0, len(items[0])], [len(x) for x in items], opts, 4, 0, d_out, [0, caps[0]], caps)
        back = bytearray(sum(caps))
        ctx.d2h(back, d_out, sum(caps))
        assert got == [(OK, len(want[0])), (OK, len(want[1]))]
        assert bytes(back[: got[0][1]]) == want[0] and bytes(back[caps[0]: caps[0] + got[1][1]]) == want[1]
        assert ctx.stream_encode_batch_device(d_in, [], [], opts, 4, 0, d_out, [], []) == []
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    assert ctx.stream_encode_batch([], preset=0) == []
    assert xz_b200.stream_bound(5, 0) == 0


def test_call_level_errors(ctx):
    import xz_b200
    for kw, code in (({"block_size": (1 << 30) + 1}, OPTIONS_ERROR), ({"check": 2}, UNSUPPORTED_CHECK)):
        with pytest.raises(xz_b200.XzError) as e:
            ctx.stream_encode_batch([b"abc", b""], preset=1, caps=[4096, 4096], **kw)
        assert e.value.code == code
