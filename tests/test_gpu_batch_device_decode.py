"""GPU tests (-m gpu) of xzb_stream_buffer_decode_batch_device: Streams and output slots in device memory, the container
read on the GPU.  Per item the call gives what the host batch gives -- (ret, out_size, in_used) and the slot's first
out_size bytes -- over the reference's decoder corpus, the recorded lzma_stream_buffer_decode cases and a mixed batch
(all four checks, Delta / BCJ chains, sized and unsized Blocks, empty items, odd offsets, adjacent slots).  A pattern
written around and into the slots shows that nothing outside a slot changes, nor anything past out_size of an item that
decoded.  Encode-then-decode from device memory gives every item back, and the call copies no item data."""
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
MiB = 1 << 20
PAT = 0x5A


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


def dev_decode(ctx, streams, caps, flags=0, in_gap=0, out_gap=0):
    """Device batch decode with item i at an odd offset of d_in and slot i at an odd offset of d_out, out_gap bytes after
    slot i - 1 (0: adjacent).  Returns [(ret, slot[:out_size], in_used)] after checking the pattern around the slots."""
    n = len(streams)
    in_off, pos = [], 1
    for s in streams:
        in_off.append(pos); pos += len(s) + in_gap
    out_off, opos = [], 3
    for c in caps:
        out_off.append(opos); opos += c + out_gap
    opos += 5
    src = bytearray(pos)
    for o, s in zip(in_off, streams):
        src[o:o + len(s)] = s
    d_in, d_out = ctx.device_alloc(len(src)), ctx.device_alloc(opos)
    try:
        ctx.h2d(d_in, bytes(src), len(src))
        ctx.h2d(d_out, bytes([PAT]) * opos, opos)
        res = ctx.stream_buffer_decode_batch_device(d_in, in_off, [len(s) for s in streams], d_out, out_off, caps, flags)
        back = bytearray(opos)
        ctx.d2h(back, d_out, opos)
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    assert len(res) == n
    inside = bytearray(opos)
    for o, c in zip(out_off, caps):
        inside[o:o + c] = b"\x01" * c
    outside = bytes(b for b, m in zip(back, inside) if not m)
    assert outside == bytes([PAT]) * len(outside), "a byte outside every slot changed"
    got = []
    for o, c, (r, size, used) in zip(out_off, caps, res):
        assert size <= c
        if r == 0:
            assert back[o + size:o + c] == bytes([PAT]) * (c - size), "bytes past out_size changed in a slot that decoded"
        got.append((r, bytes(back[o:o + size]), used))
    return got


def test_corpus_equals_host_batch(ctx):
    """All of the reference's decoder corpus (Delta, x86 and ARM64 chains included) as one device batch."""
    names = sorted(os.listdir(os.path.join(GOLD, "ref_files")))
    files = [open(os.path.join(GOLD, "ref_files", f), "rb").read() for f in names]
    caps = [1 << 20] * len(files)
    want = ctx.stream_buffer_decode_batch(files, caps)
    got = dev_decode(ctx, files, caps)
    for name, w, g in zip(names, want, got):
        assert g == w, name
    verdicts = json.load(open(os.path.join(GOLD, "decode_verdicts.json")))
    for name, (r, out, _) in zip(names, got):
        if name in verdicts:
            v = verdicts[name]
            assert r == (9 if v["ret"] == 10 else v["ret"]) and len(out) == v["out_size"], name   # truncated input: LZMA_DATA_ERROR here


def test_recorded_cases_equal_host_batch_and_reference(ctx):
    import make_golden as MG
    g = json.load(open(os.path.join(GOLD, "buffer_golden.json")))["decode"]
    enc, by_flags = {}, {}
    for name, kind, preset, n, m in MG.buffer_decode_cases():
        key = (kind, preset, n, m[0] == "nocheck")
        if key not in enc:
            enc[key] = X.oracle_buffer_encode(X.gendata(kind, n), n, preset, 0 if key[3] else 4)
        data, cap, flags = MG.buffer_apply(enc[key], n, m)
        by_flags.setdefault(flags, []).append((name, data, cap))
    for flags, group in sorted(by_flags.items()):
        xflags = 2 if flags & 0x10 else 0
        want = ctx.stream_buffer_decode_batch([d for _, d, _ in group], [c for _, _, c in group], xflags)
        got = dev_decode(ctx, [d for _, d, _ in group], [c for _, _, c in group], xflags, in_gap=2)
        for (name, _, _), w, (r, out, used) in zip(group, want, got):
            assert (r, out, used) == w, name
            if (flags & ~0x30) == 0 and r == 0:
                v = g[name]
                assert (r, used, len(out), hashlib.sha256(out).hexdigest()) == (v["ret"], v["in_used"], v["out_size"], v["out_sha256"]), name


def test_mixed_batch(ctx):
    """Checks None / CRC32 / CRC64 / SHA-256, Delta and BCJ chains from set_filters, sized and unsized Blocks, empty items,
    a slot one byte short, a cut Stream; odd offsets and adjacent slots; n = 0."""
    rng = random.Random(21)
    streams, caps, items = [], [], []
    chains = ([], [(0x03, 4)], [(0x04, 0)], [(0x03, 1), (0x07, 0)])
    for i in range(48):
        n = rng.choice((0, 1, 3000, 65536, 150001, 400000))
        x = bytes(X.gendata("TER"[i % 3], n)[:n])
        check = (0, 1, 4, 10)[i % 4]
        ctx.set_filters(chains[(i // 4) % 4])
        try:
            if i % 3 == 0:
                s = ctx.stream_encode(x, preset=1, block_size=1 << 16, check=check) if n else ctx.stream_buffer_encode(x, check=check)
            else:
                s = ctx.stream_buffer_encode(x, preset=1 + i % 6, check=check)
        finally:
            ctx.set_filters([])
        if i % 5 == 1 and n:
            s = X.drop_block_sizes(s)
        cap = n
        if i % 11 == 3 and n:
            cap = n - 1
        if i % 13 == 5 and n:
            s = s[:-17]
        streams.append(s); caps.append(cap); items.append(x)
    streams += [b"", b"\xfd7zXZ"]
    caps += [0, 10]
    items += [b"", b""]
    want = ctx.stream_buffer_decode_batch(streams, caps)
    got = dev_decode(ctx, streams, caps, in_gap=1)
    assert got == want
    ok = [r == 0 for r, _, _ in got]
    assert sum(ok) > 30 and not all(ok)
    for (r, out, _), x in zip(got, items):
        if r == 0:
            assert out == x
    assert ctx.stream_buffer_decode_batch_device(0, [], [], 0, [], [], 0) == []


@pytest.mark.parametrize("preset", [1, 6])
def test_device_round_trip(ctx, preset):
    """300 seeded items of up to 3 MiB: the device encode batch, then the device decode batch of its output, all in HBM;
    only the final comparison reads the decoded bytes back."""
    import xz_b200
    rng = random.Random(100 + preset)
    top = 3 * MiB
    sizes = [0, 1, top] + [int(top ** rng.random()) for _ in range(297)]
    rng.shuffle(sizes)
    items = [bytes(X.gendata("TER"[i % 3], s)[:s]) for i, s in enumerate(sizes)]
    in_off, pos = [], 0
    for x in items:
        in_off.append(pos); pos += len(x)
    src = b"".join(items)
    caps = [xz_b200.lib().xzb_stream_buffer_bound(len(x)) for x in items]
    enc_off, epos = [], 0
    for c in caps:
        enc_off.append(epos); epos += c
    dec_off, dpos = [], 0
    for x in items:
        dec_off.append(dpos); dpos += len(x)
    d_src, d_xz, d_back = ctx.device_alloc(max(pos, 1)), ctx.device_alloc(epos), ctx.device_alloc(max(dpos, 1))
    try:
        ctx.h2d(d_src, src, len(src))
        enc = ctx.stream_buffer_encode_batch_device(d_src, in_off, sizes, xz_b200.lzma_lzma_preset(preset), 4, d_xz, enc_off, caps)
        assert [r for r, _ in enc] == [0] * len(items)
        dec = ctx.stream_buffer_decode_batch_device(d_xz, enc_off, [s for _, s in enc], d_back, dec_off, sizes)
        st = ctx.stats()
        assert st.ms_h2d == 0 and st.ms_d2h == 0 and st.n_blocks == sum(1 for s in sizes if s)
        assert st.n_positions == sum(sizes)
        back = bytearray(max(dpos, 1))
        ctx.d2h(back, d_back, dpos)
    finally:
        ctx.device_free(d_src); ctx.device_free(d_xz); ctx.device_free(d_back)
    assert dec == [(0, n, xz_size) for n, (_, xz_size) in zip(sizes, enc)]
    assert bytes(back[:dpos]) == src
