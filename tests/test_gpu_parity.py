"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI (libxzb200.so), against
the oracle on the same seeded inputs, against the committed golden vectors produced by the
unmodified reference, and -- at sizes the oracle cannot finish quickly -- through
size-independent properties (decode(encode(x)) == x by the GPU *and* by the oracle decoder,
Index records consistent with the bytes)."""
import ctypes as C
import hashlib
import json
import os

import pytest

import xzlibs as X

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MiB = 1 << 20


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


def _golden(max_size, min_size=0):
    cases = json.load(open(os.path.join(GOLD, "encode_golden.json")))
    return [c for c in cases if min_size <= c["size"] <= max_size]


@pytest.mark.parametrize("case", _golden(300000), ids=lambda c: f"{c['kind']}-{c['preset']:#x}-{c['size']}")
def test_encode_matches_reference_golden_small(ctx, case):
    """Edge sizes 0..300000 (empty, 1-5 bytes, 273, 4096, 65535/6/7) x presets 0,1,3,4,6,9e x T/E/R."""
    n = case["size"]
    buf = X.gendata(case["kind"], n)
    out = ctx.stream_encode(buf, preset=case["preset"], block_size=case["block_size"], check=case["check"], n=n)
    assert len(out) == case["xz_size"]
    assert hashlib.sha256(out).hexdigest() == case["xz_sha256"]
    r, back = ctx.stream_decode(out, n)
    assert r == 0 and back == bytes(buf[:n])


@pytest.mark.parametrize("case", _golden(4 * MiB, 300001), ids=lambda c: f"{c['kind']}-{c['preset']:#x}-{c['size']}-{c['block_size']}")
def test_encode_matches_reference_golden_chunk_and_block_edges(ctx, case):
    """2 MiB +- 273 (LZMA2 chunk limit), multi-block streams with a short last block."""
    n = case["size"]
    buf = X.gendata(case["kind"], n)
    out = ctx.stream_encode(buf, preset=case["preset"], block_size=case["block_size"], check=case["check"], n=n)
    assert hashlib.sha256(out).hexdigest() == case["xz_sha256"]


@pytest.mark.parametrize("kind,preset", [("T", 1), ("R", 3)])
def test_encode_full_block_fast_presets_golden(ctx, kind, preset):
    """One full 16 MiB block at the BASELINE block size: config 0 (-1, T) and config 4's
    incompressible case (-3, R: every chunk raw, block lands exactly on lzma_block_buffer_bound)."""
    case = [c for c in _golden(16 * MiB, 16 * MiB) if c["kind"] == kind and c["preset"] == preset and c["size"] == 16 * MiB][0]
    buf = X.gendata(kind, case["size"])
    out = ctx.stream_encode(buf, preset=preset, block_size=case["block_size"], n=case["size"])
    assert len(out) == case["xz_size"] and hashlib.sha256(out).hexdigest() == case["xz_sha256"]
    r, back = ctx.stream_decode(out, case["size"])
    assert r == 0 and back == bytes(buf[: case["size"]])


@pytest.mark.parametrize("kind,preset,size", [("T", 6, 16 * MiB), ("T", 6, 16 * MiB + 1), ("E", 6, 16 * MiB), ("E", 9 | X.XZ_PRESET_EXTREME, 4 * MiB)])
def test_encode_full_block_normal_mode_golden(ctx, kind, preset, size):
    """BASELINE's own block size (16 MiB) at -6 / -9e: SHA-256 of the GPU stream == the unmodified
    reference's (golden), incl. the 16 MiB + 1 byte case (a full Block plus a 1-byte Block)."""
    case = [c for c in _golden(17 * MiB, 4 * MiB) if c["kind"] == kind and c["preset"] == preset and c["size"] == size][0]
    buf = X.gendata(kind, size)
    out = ctx.stream_encode(buf, preset=preset, block_size=case["block_size"], n=size)
    assert len(out) == case["xz_size"] and hashlib.sha256(out).hexdigest() == case["xz_sha256"]
    r, back = ctx.stream_decode(out, size)
    assert r == 0 and back == bytes(buf[:size])


def test_config4_block_shape_9e_16MiB_golden(ctx):
    """BASELINE configs[3]'s real Block shape: 16 MiB of `E` at -9e (bt4, nice 273, depth 512, 64 MiB dict).  Two Blocks,
    each compared with the per-Block SHA-256 recorded from the unmodified reference (tests/golden/bench_golden.json)."""
    gold = json.load(open(os.path.join(GOLD, "bench_golden.json")))["E9e"]
    bs, nb = gold["block_size"], 2
    n = nb * bs
    buf = X.gendata("E", n)
    out = ctx.stream_encode(buf, preset=gold["preset"], block_size=bs, n=n)
    pos = 12
    for i in range(nb):
        total, sha = gold["blocks"][i]
        assert hashlib.sha256(out[pos:pos + total]).hexdigest() == sha, f"Block {i}"
        pos += total
    r, back = ctx.stream_decode(out, n)
    assert r == 0 and back == bytes(buf[:n])


def test_encode_vs_oracle_all_match_finders_and_lclppb(ctx):
    import xz_b200
    n = 200000
    buf = X.gendata("T", n)
    for mode in (1, 2):
        for mf in (0x03, 0x04, 0x12, 0x13, 0x14):
            for lc, lp, pb in ((3, 0, 2), (0, 2, 0), (4, 0, 4), (1, 3, 1)):
                o = X.LzmaOptions(1 << 16, lc, lp, pb, mode, 48, mf, 0)
                po = xz_b200.LzmaOptions(1 << 16, lc, lp, pb, mode, 48, mf, 0)
                assert ctx.stream_encode(buf, opts=po, block_size=1 << 17, n=n) == X.oracle_encode(buf, n, 0, 1 << 17, opts=o)


def test_check_types(ctx):
    n = 70000
    buf = X.gendata("E", n)
    for check in (X.CHECK_NONE, X.CHECK_CRC32, X.CHECK_CRC64):
        out = ctx.stream_encode(buf, preset=1, block_size=1 << 16, check=check, n=n)
        assert out == X.oracle_encode(buf, n, 1, 1 << 16, check=check)
        r, back = ctx.stream_decode(out, n)
        assert r == 0 and back == bytes(buf[:n])


def test_decoder_corpus_verdicts(ctx):
    """The reference's own decoder fixtures (tests/files/*.xz): same lzma_ret and same bytes."""
    verdicts = json.load(open(os.path.join(GOLD, "decode_verdicts.json")))
    n = 0
    for name, v in sorted(verdicts.items()):   # incl. the files with Delta / ARM64 / x86 filters in front of LZMA2
        data = open(os.path.join(GOLD, "ref_files", name), "rb").read()
        r, out = ctx.stream_decode(data, 1 << 20)
        assert r == v["ret"], (name, r, v["ret"])
        assert len(out) == v["out_size"], name  # also on errors: what was decoded before the error is delivered
        if r == 0:
            assert hashlib.sha256(out).hexdigest() == v["out_sha256"], name
        n += 1
    assert n > 50


def test_truncated_and_corrupt(ctx):
    n = 50000
    buf = X.gendata("T", n)
    xz = X.oracle_encode(buf, n, 6, 1 << 14)
    for cut in (0, 5, 11, 12, 13, 40, len(xz) // 2, len(xz) - 1):
        assert ctx.stream_decode(xz[:cut], n)[0] == X.oracle_decode(xz[:cut], n)[0] == 10
    for where in (len(xz) // 3, len(xz) // 2, len(xz) - 20):
        bad = bytearray(xz)
        bad[where] ^= 0x55
        assert ctx.stream_decode(bytes(bad), n)[0] == X.oracle_decode(bytes(bad), n)[0]


def test_device_block_api_and_index_records(ctx):
    """xzb_encode_blocks_device: Blocks back to back + Index records; reassembling the Stream
    from them gives the oracle's bytes (this is what each rank does before the index gather)."""
    import xz_b200
    n, bs = 5 * MiB // 2 + 17, 1 * MiB
    buf = X.gendata("E", n)
    o = xz_b200.lzma_lzma_preset(1)
    d_in = ctx.device_alloc(n)
    cap = 3 * xz_b200.lzma_block_buffer_bound(bs)
    d_out = ctx.device_alloc(cap)
    ctx.h2d(d_in, buf, n)
    size, recs = ctx.encode_blocks_device(d_in, n, o, 4, bs, d_out, cap)
    host = (C.c_uint8 * size)()
    ctx.d2h(host, d_out, size)
    idx = xz_b200.index_encode(recs)
    stream = xz_b200.stream_header(4) + bytes(host) + idx + xz_b200.stream_footer(4, len(idx))
    assert stream == X.oracle_encode(buf, n, 1, bs)
    assert sum((u + 3) // 4 * 4 for u, _ in recs) == size and sum(v for _, v in recs) == n
    # device-resident decode of the same blocks
    offs, comp, unc, ooff, pos, opos = [], [], [], [], 0, 0
    for u, v in recs:
        hs = (host[pos] + 1) * 4
        offs.append(pos + hs); comp.append(u - hs - 8); unc.append(v); ooff.append(opos)
        pos += (u + 3) // 4 * 4; opos += v
    d_back = ctx.device_alloc(n)
    rets, crcs = ctx.decode_blocks_device(d_out, offs, comp, unc, ooff, [o.dict_size] * len(recs), 4, d_back)
    assert rets == [0] * len(recs)
    back = (C.c_uint8 * n)()
    ctx.d2h(back, d_back, n)
    assert bytes(back) == bytes(buf[:n])
    for i, (u, v) in enumerate(recs):
        assert crcs[i] == X.oracle().xzo_crc64(bytes(buf[ooff[i]:ooff[i] + v]), v, 0)
    for p in (d_in, d_out, d_back):
        ctx.device_free(p)


@pytest.mark.parametrize("kind", "TE")
def test_normal_mode_multi_block_properties(ctx, kind):
    """-6 on 8 x 1 MiB blocks: bytes equal the oracle's, and the round trip holds through both
    the GPU decoder and the oracle decoder."""
    n, bs = 8 * MiB, 1 * MiB
    buf = X.gendata(kind, n)
    out = ctx.stream_encode(buf, preset=6, block_size=bs, n=n)
    assert hashlib.sha256(out).hexdigest() == hashlib.sha256(X.oracle_encode(buf, n, 6, bs)).hexdigest()
    r, back = ctx.stream_decode(out, n)
    assert r == 0 and back == bytes(buf[:n])
    r, back = X.oracle_decode(out, n)
    assert r == 0 and back == bytes(buf[:n])


def test_multiple_waves_give_the_same_bytes(monkeypatch):
    """Streams longer than one wave are encoded wave by wave (XZB_MAX_WAVE_BLOCKS forces 2-block waves
    here); bytes must not depend on the wave size."""
    import xz_b200
    n, bs = 5 * 262144 + 1234, 262144
    buf = X.gendata("E", n)
    want = X.oracle_encode(buf, n, 6, bs)
    monkeypatch.setenv("XZB_MAX_WAVE_BLOCKS", "2")
    c = xz_b200.Context(0)
    try:
        assert c.stream_encode(buf, preset=6, block_size=bs, n=n) == want
        assert c.stats().n_blocks == 6
    finally:
        c.close()


def test_fast_mode_kernel_forms_match_oracle(ctx):
    """Fast mode (presets 0-3) runs in one of two launch forms, chosen per wave: a wave with more Blocks than
    the GPU has SMs (400 here, more than any H100 has) packs several Blocks per SM with a coder warp for the
    range coder; a wave of a few Blocks gives every Block an SM to itself.  Both must give the oracle's bytes,
    for hash chains (presets 1 and 3) and for a binary tree (BT4)."""
    import xz_b200
    bt4 = xz_b200.lzma_lzma_preset(2)
    bt4.mf, bt4.nice_len, bt4.depth = 0x14, 64, 0
    xbt4 = X.preset_options(2); xbt4.mf, xbt4.nice_len, xbt4.depth = 0x14, 64, 0
    for nblocks, bs in ((400, 4096), (3, 1 << 17)):
        n = nblocks * bs - 123   # short last Block
        for kind, preset in (("T", 1), ("R", 1), ("T", 3), ("R", 3)):
            buf = X.gendata(kind, n)
            assert ctx.stream_encode(buf, preset=preset, block_size=bs, n=n) == X.oracle_encode(buf, n, preset, bs), (nblocks, kind, preset)
        buf = X.gendata("T", n)
        assert ctx.stream_encode(buf, opts=bt4, block_size=bs, n=n) == X.oracle_encode(buf, n, 2, bs, opts=xbt4), (nblocks, "bt4")
        assert ctx.stats().n_blocks == nblocks


@pytest.mark.parametrize("seg_shift,overlap", [(8, 1), (10, 1), (12, 0), (16, 1), (20, 0)])
def test_match_finder_segments_and_overlap_do_not_change_bytes(monkeypatch, seg_shift, overlap):
    """The binary-tree match finder works through every block in segments of 2^XZB_SEG_SHIFT positions and
    the parser kernel consumes finished segments while later ones are still being searched
    (XZB_OVERLAP=0 runs them back to back).  Neither knob may change a byte."""
    import xz_b200
    monkeypatch.setenv("XZB_SEG_SHIFT", str(seg_shift))
    monkeypatch.setenv("XZB_OVERLAP", str(overlap))
    c = xz_b200.Context(0)
    try:
        for kind, preset, n, bs in (("T", 6, 3 * 400000 + 17, 400000), ("E", 6, 700000, 1 << 20), ("R", 5, 300000, 1 << 17),
                                    ("L", 9 | X.XZ_PRESET_EXTREME, 500000, 1 << 19), ("T", 4, 4, 1 << 16), ("T", 6, 0, 1 << 16)):
            buf = X.gendata(kind, n)
            assert c.stream_encode(buf, preset=preset, block_size=bs, n=n) == X.oracle_encode(buf, n, preset, bs), (kind, preset, n)
        o = xz_b200.lzma_lzma_preset(2)  # fast mode on a binary tree: only the front warp runs, same polling
        o.mf, o.nice_len, o.depth = 0x14, 64, 0
        xo = X.preset_options(2); xo.mf, xo.nice_len, xo.depth = 0x14, 64, 0
        buf = X.gendata("T", 600000)
        assert c.stream_encode(buf, opts=o, block_size=1 << 18, n=600000) == X.oracle_encode(buf, 600000, 2, 1 << 18, opts=xo)
    finally:
        c.close()


@pytest.mark.parametrize("preset", [1, 6])
def test_sha256_check_encode_and_verify(ctx, preset):
    """LZMA_CHECK_SHA256: the Check field of every Block equals the oracle's (== reference's) bytes, the decoder
    verifies it (a flipped digest byte is LZMA_DATA_ERROR, and LZMA_IGNORE_CHECK semantics via the flag)."""
    n, bs = 3 * 300000 + 5, 300000
    buf = X.gendata("T", n)
    xz = ctx.stream_encode(buf, preset=preset, block_size=bs, check=10, n=n)
    assert xz == X.oracle_encode(buf, n, preset, bs, check=10)
    r, back = ctx.stream_decode(xz, n)
    assert r == 0 and back == bytes(buf[:n])
    hsize = (xz[12] + 1) * 4
    # first Block: header, data (compressed size from the Index is not needed: flip a byte of the LAST Block's digest)
    idx_size = (int.from_bytes(xz[-8:-4], "little") + 1) * 4
    digest_end = len(xz) - 12 - idx_size
    bad = bytearray(xz); bad[digest_end - 7] ^= 0x20
    r, _ = ctx.stream_decode(bytes(bad), n)
    assert r == 9
    r, back, used = ctx.stream_buffer_decode(bytes(bad), n, flags=2)  # XZB_DEC_IGNORE_CHECK
    assert r == 0 and back == bytes(buf[:n]) and used == len(bad) and hsize > 0
