"""The encoder kernels on Blocks that switch between LZMA and uncompressed LZMA2 chunks (-m gpu).

Every case of tests/chunk_mix.py must encode to the reference's Stream (the chunk_mix section of
tests/golden/ref_live_golden.json), with the oracle's LZMA / uncompressed chunk counts, and decode back through
stream_decode and stream_buffer_decode_batch_device.  A wrong state after an uncompressed chunk (probabilities, reps,
price counters, pending symbols, the fast parser's restart, pos_state after swallowed read_ahead bytes) still
decodes, so only the byte comparison catches it.  The one-shot items, whose LZMA2 data ends a few bytes either side of
lzma2_bound, go through both batch encode calls."""

import pytest

import chunk_mix as M
import xzlibs as X

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


def _as_product(o):
    import xz_b200
    return xz_b200.LzmaOptions(*[getattr(o, f) for f, _ in X.LzmaOptions._fields_])


def _gold(case):
    return X.ref_golden()["chunk_mix"][M.key(case)]


_streams = {}


@pytest.mark.parametrize("i", range(len(M.cases())), ids=[c.name for c in M.cases()])
def test_encode_identical_with_the_reference_chunks(ctx, i):
    case = M.cases()[i]
    xz = ctx.stream_encode(case.data, block_size=case.block_size, check=case.check, opts=_as_product(case.opts))
    st = ctx.stats()
    assert X.sha64(xz) == _gold(case)["stream"], M.key(case)
    assert [st.n_chunks_lzma, st.n_chunks_raw] == _gold(case)["chunks"], M.key(case)
    r, back = ctx.stream_decode(xz, len(case.data))
    assert r == 0 and back == case.data, M.key(case)
    _streams[case.name] = xz


def test_device_batch_decode_gives_every_input_back(ctx):
    cases = M.cases()
    streams = [_streams.get(c.name) or ctx.stream_encode(c.data, block_size=c.block_size, check=c.check, opts=_as_product(c.opts))
               for c in cases]
    in_off, pos = [], 0
    for s in streams:
        in_off.append(pos); pos += len(s)
    out_off, opos = [], 0
    for c in cases:
        out_off.append(opos); opos += len(c.data)
    d_in, d_out = ctx.device_alloc(pos), ctx.device_alloc(opos)
    try:
        ctx.h2d(d_in, b"".join(streams), pos)
        res = ctx.stream_buffer_decode_batch_device(d_in, in_off, [len(s) for s in streams], d_out, out_off, [len(c.data) for c in cases])
        back = bytearray(opos)
        ctx.d2h(back, d_out, opos)
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    for c, s, o, r in zip(cases, streams, out_off, res):
        assert r == (0, len(c.data), len(s)) and bytes(back[o:o + len(c.data)]) == c.data, c.name


@pytest.mark.parametrize("preset", [0, 6])
def test_oneshot_items_near_the_bound_in_both_batch_calls(ctx, preset):
    """Items whose LZMA2 data is 3 bytes under to 2 bytes over lzma2_bound(n): the Block keeps the LZMA2 data or falls
    back to an uncompressed Block as lzma_easy_buffer_encode does, from host and from device memory."""
    import xz_b200
    items = [(name, data) for name, p, data in M.oneshot_items() if p == preset]
    assert len(items) == 6
    o = xz_b200.lzma_lzma_preset(preset)
    want = [X.ref_golden()["chunk_mix"][name]["stream"] for name, _ in items]
    got = ctx.stream_buffer_encode_batch([d for _, d in items], check=X.CHECK_CRC64, opts=o)
    assert [(r, X.sha64(s)) for r, s in got] == [(0, w) for w in want]
    sizes = [len(d) for _, d in items]
    caps = [xz_b200.lib().xzb_stream_buffer_bound(n) for n in sizes]
    in_off = [sum(sizes[:k]) for k in range(len(items))]
    out_off = [sum(caps[:k]) for k in range(len(items))]
    d_in, d_out = ctx.device_alloc(sum(sizes)), ctx.device_alloc(sum(caps))
    try:
        ctx.h2d(d_in, b"".join(d for _, d in items), sum(sizes))
        res = ctx.stream_buffer_encode_batch_device(d_in, in_off, sizes, o, X.CHECK_CRC64, d_out, out_off, caps)
        out = bytearray(sum(caps))
        ctx.d2h(out, d_out, len(out))
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    assert [r for r, _ in res] == [0] * len(items)
    assert [X.sha64(out[off:off + sz]) for off, (_, sz) in zip(out_off, res)] == want


def test_serial_small_segments_and_small_waves_give_the_same_bytes(monkeypatch):
    """One normal-mode case with the match finder and the parser serialised (XZB_OVERLAP=0), 1 KiB match-finder
    segments (XZB_SEG_SHIFT=10) and at most 2 Blocks per wave (XZB_MAX_WAVE_BLOCKS=2)."""
    import xz_b200
    monkeypatch.setenv("XZB_OVERLAP", "0")
    monkeypatch.setenv("XZB_SEG_SHIFT", "10")
    monkeypatch.setenv("XZB_MAX_WAVE_BLOCKS", "2")
    case = [c for c in M.cases() if c.name == "preset-6"][0]
    c = xz_b200.Context(0)
    try:
        xz = c.stream_encode(case.data, block_size=case.block_size, check=case.check, opts=_as_product(case.opts))
        assert X.sha64(xz) == _gold(case)["stream"]
        assert [c.stats().n_chunks_lzma, c.stats().n_chunks_raw] == _gold(case)["chunks"]
    finally:
        c.close()
