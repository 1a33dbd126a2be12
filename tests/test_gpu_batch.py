"""GPU tests (-m gpu) of the batch one-shot calls (xzb_stream_buffer_encode_batch[_device], xzb_stream_buffer_decode_batch):
every item of a batch gets what the single call gives it alone -- the reference's bytes (tests/golden/buffer_golden.json)
for the recorded one-shot Streams, the single call's bytes for seeded batches of mixed sizes in one wave and in many,
with a BCJ chain, from device memory and with an output slot one byte short -- and a batch of Streams decodes item by
item as the single decoder does, the reference's verdicts included."""
import hashlib
import json
import os
import random
import sys

import pytest

import xzlibs as X

pytestmark = pytest.mark.gpu
GOLD = os.path.join(X.ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
BUF_ERROR = 10
MiB = 1 << 20


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


def _data(kind, n):
    return bytes(X.gendata(kind, n)[:n])


def test_encode_batches_match_reference_golden(ctx):
    """The recorded one-shot Streams, one batch per (preset, check), shuffled, with one item twice: sizes 0 to 16 MiB in
    one wave, fast and normal mode, -9e."""
    cases = json.load(open(os.path.join(GOLD, "buffer_golden.json")))["encode"]
    groups = {}
    for c in cases:
        groups.setdefault((c["preset"], c["check"]), []).append(c)
    assert sum(len(g) for g in groups.values()) == 211
    rng = random.Random(11)
    for (preset, check), g in sorted(groups.items()):
        g = g + [g[len(g) // 2]]
        rng.shuffle(g)
        out = ctx.stream_buffer_encode_batch([_data(c["kind"], c["size"]) for c in g], preset=preset, check=check)
        for c, (r, xz) in zip(g, out):
            assert r == 0 and len(xz) == c["xz_size"] and hashlib.sha256(xz).hexdigest() == c["xz_sha256"], (preset, check, c["kind"], c["size"])


def _seeded_items(seed, count=300, top=3 * MiB):
    """Sizes 0 .. 3 MiB, log-uniform (so most are small, as filesystem blocks are), 0, 1 and 3 MiB included."""
    rng = random.Random(seed)
    sizes = [0, 1, top] + [int(top ** rng.random()) for _ in range(count - 3)]
    rng.shuffle(sizes)
    kinds = "TER"
    return [_data(kinds[i % 3], s) for i, s in enumerate(sizes)]


@pytest.mark.parametrize("preset", [1, 6])
def test_seeded_batch_equals_single_calls_in_one_wave_and_many(ctx, monkeypatch, preset):
    """~300 items: the batch equals stream_buffer_encode of each item alone.  At -1 the wave has more Blocks than SMs
    (the coder-warp form of the fast parser); XZB_MAX_WAVE_BLOCKS=7 spreads the same batch over many waves."""
    import xz_b200
    items = _seeded_items(preset)
    want = [ctx.stream_buffer_encode(x, preset=preset) for x in items]
    got = ctx.stream_buffer_encode_batch(items, preset=preset)
    assert [r for r, _ in got] == [0] * len(items)
    assert [xz for _, xz in got] == want
    non_empty = sum(1 for x in items if x)
    assert ctx.stats().n_blocks == non_empty
    monkeypatch.setenv("XZB_MAX_WAVE_BLOCKS", "7")
    c7 = xz_b200.Context(0)
    try:
        got7 = c7.stream_buffer_encode_batch(items, preset=preset)
        assert [xz for _, xz in got7] == want and [r for r, _ in got7] == [0] * len(items)
    finally:
        c7.close()


def test_bcj_chain_device_variant_and_short_slot(ctx):
    """An x86 BCJ filter on the context applies to every item; the device form writes the host form's bytes; an item
    whose slot is one byte short gets XZB_BUF_ERROR and its neighbours are unaffected."""
    import xz_b200
    items = [_data("E", n) for n in (70000, 0, 5, 300001, 4096, 131072, 65537)]
    ctx.set_filters([(0x04, 0)])
    try:
        want = [ctx.stream_buffer_encode(x, preset=6) for x in items]
        got = ctx.stream_buffer_encode_batch(items, preset=6)
        assert [r for r, _ in got] == [0] * len(items) and [xz for _, xz in got] == want
    finally:
        ctx.set_filters([])
    want = [ctx.stream_buffer_encode(x, preset=3, check=1) for x in items]
    caps = [len(w) for w in want]
    caps[3] -= 1
    got = ctx.stream_buffer_encode_batch(items, preset=3, check=1, caps=caps)
    assert [r for r, _ in got] == [0, 0, 0, BUF_ERROR, 0, 0, 0]
    assert [xz for i, (_, xz) in enumerate(got) if i != 3] == [w for i, w in enumerate(want) if i != 3] and got[3][1] == b""
    # device memory: inputs and slots at odd offsets
    in_off, pos = [], 3
    for x in items:
        in_off.append(pos); pos += len(x) + 5
    src = bytearray(pos)
    for o, x in zip(in_off, items):
        src[o:o + len(x)] = x
    caps = [xz_b200.lib().xzb_stream_buffer_bound(len(x)) for x in items]
    out_off, opos = [], 1
    for c in caps:
        out_off.append(opos); opos += c + 3
    d_in, d_out = ctx.device_alloc(len(src)), ctx.device_alloc(opos)
    try:
        ctx.h2d(d_in, bytes(src), len(src))
        res = ctx.stream_buffer_encode_batch_device(d_in, in_off, [len(x) for x in items], xz_b200.lzma_lzma_preset(3), 1, d_out, out_off, caps)
        back = bytearray(opos)
        ctx.d2h(back, d_out, opos)
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    assert [r for r, _ in res] == [0] * len(items)
    assert [bytes(back[o:o + s]) for o, (_, s) in zip(out_off, res)] == want


def test_decode_batches_match_single_calls_and_reference_verdicts(ctx):
    """The recorded lzma_stream_buffer_decode cases, one batch per flags value: per item (ret, bytes, in_used) of the
    single call; without LZMA_CONCATENATED / LZMA_TELL_* (which the liblzma-named wrapper handles around these calls)
    and without the flag that wrapper rejects, the reference's verdict too."""
    import make_golden as MG
    g = json.load(open(os.path.join(GOLD, "buffer_golden.json")))["decode"]
    cases = MG.buffer_decode_cases()
    assert len(cases) == len(g)
    enc = {}
    by_flags = {}
    for name, kind, preset, n, m in cases:
        key = (kind, preset, n, m[0] == "nocheck")
        if key not in enc:
            enc[key] = X.oracle_buffer_encode(X.gendata(kind, n), n, preset, 0 if key[3] else 4)
        data, cap, flags = MG.buffer_apply(enc[key], n, m)
        by_flags.setdefault(flags, []).append((name, data, cap))
    for flags, group in sorted(by_flags.items()):
        xflags = 2 if flags & 0x10 else 0  # LZMA_IGNORE_CHECK -> XZB_DEC_IGNORE_CHECK
        got = ctx.stream_buffer_decode_batch([d for _, d, _ in group], [c for _, _, c in group], xflags)
        for (name, data, cap), (r, out, used) in zip(group, got):
            assert (r, out, used) == ctx.stream_buffer_decode(data, cap, xflags), name
            if (flags & ~0x30) == 0:  # none but LZMA_IGNORE_CHECK / LZMA_FAIL_FAST
                want = g[name]
                assert r == want["ret"], name
                if r == 0:
                    assert (used, len(out), hashlib.sha256(out).hexdigest()) == (want["in_used"], want["out_size"], want["out_sha256"]), name


def test_decode_batch_of_corpus_and_unsized_blocks(ctx):
    """All of tests/golden/ref_files as one batch equals the single calls; so does a batch that mixes Streams whose
    Blocks carry no sizes (decoded a Block at a time) with sized ones; batch encode then batch decode gives every item back."""
    names = sorted(os.listdir(os.path.join(GOLD, "ref_files")))
    files = [open(os.path.join(GOLD, "ref_files", f), "rb").read() for f in names]
    caps = [1 << 20] * len(files)
    got = ctx.stream_buffer_decode_batch(files, caps)
    for name, data, cap, res in zip(names, files, caps, got):
        assert res == ctx.stream_buffer_decode(data, cap), name
    items = _seeded_items(5, count=40, top=MiB)
    streams = []
    for i, x in enumerate(items):
        if i % 3 == 0:
            streams.append(X.drop_block_sizes(ctx.stream_encode(x, preset=1, block_size=1 << 16)) if x else ctx.stream_buffer_encode(x))
        elif i % 3 == 1:
            streams.append(X.drop_block_sizes(ctx.stream_buffer_encode(x, preset=1)) if x else ctx.stream_buffer_encode(x))
        else:
            streams.append(ctx.stream_encode(x, preset=1, block_size=1 << 17) if x else ctx.stream_buffer_encode(x))
    caps = [len(x) for x in items]
    got = ctx.stream_buffer_decode_batch(streams, caps)
    for s, x, res in zip(streams, items, got):
        assert res == (0, x, len(s))
    enc = ctx.stream_buffer_encode_batch(items, preset=6, check=10)
    dec = ctx.stream_buffer_decode_batch([xz for _, xz in enc], caps)
    assert [(r, out) for r, out, _ in dec] == [(0, x) for x in items]
