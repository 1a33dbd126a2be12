"""GPU tests (-m gpu) of the LZMA2 decoder kernel on the generated Streams of tests/lzma2_gen.py (valid input an
encoder byte-identical to liblzma's never writes, and a few near misses), through every GPU decode entry point, and of
the integrity-check kernels at their slicing and padding edges.

  * xzb_decode_blocks_device on the raw payloads, all cases in one call at odd offsets: the warp form of the decoder
    (xzb_dec_warp.cuh) with exact sizes, and xzb_k_crc's CRC32 / CRC64 of what it wrote;
  * xzb_stream_decode per Stream, sized and unsized (the unsized Blocks take the grow-and-retry path);
  * xzb_stream_buffer_decode_batch and xzb_stream_buffer_decode_batch_device over all Streams as one batch;
  * xzb_k_crc at sizes around its 1023-slice split, xzb_k_sha256 at its padding boundaries, and the Check field
    verdicts of both Stream batch calls (intact, one bit flipped, flipped with XZB_DEC_IGNORE_CHECK).

Expected bytes come from the generator, which builds them by construction; the reference decoder agreed with them when
ref_live_golden.json was recorded (tests/test_lzma2_gen_cpu.py checks that record)."""
import ctypes as C
import struct
import zlib

import pytest

import lzma2_gen as G
import xzlibs as X

pytestmark = pytest.mark.gpu
MiB = 1 << 20
IGNORE_CHECK = 2      # XZB_DEC_IGNORE_CHECK


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cases():
    return G.cases()


def crc(check, data):
    return zlib.crc32(data) if check == 1 else X.oracle().xzo_crc64(data, len(data), 0)


def _odd_offsets(sizes, start):
    offs, pos = [], start
    for n in sizes:
        offs.append(pos)
        pos += n + 2 + (n & 1)      # every offset odd, a gap after each item
    return offs, pos


def decode_blocks(ctx, payloads, out_sizes, dict_sizes, check):
    """xzb_decode_blocks_device on payloads at odd offsets of one device buffer: (rets, check values, outputs)."""
    in_off, in_total = _odd_offsets([len(p) for p in payloads], 1)
    out_off, out_total = _odd_offsets(out_sizes, 3)
    src = bytearray(in_total)
    for o, p in zip(in_off, payloads):
        src[o:o + len(p)] = p
    d_in, d_out = ctx.device_alloc(in_total), ctx.device_alloc(out_total)
    try:
        ctx.h2d(d_in, bytes(src), in_total)
        rets, checks = ctx.decode_blocks_device(d_in, in_off, [len(p) for p in payloads], out_sizes, out_off, dict_sizes, check, d_out)
        back = bytearray(out_total)
        ctx.d2h(back, d_out, out_total)
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    return rets, checks, [bytes(back[o:o + n]) for o, n in zip(out_off, out_sizes)]


@pytest.mark.parametrize("check", [1, 4])
def test_decode_blocks_device_on_generated_payloads(ctx, cases, check):
    rets, checks, outs = decode_blocks(ctx, [c.payload for c in cases], [c.declared for c in cases], [c.dict_size for c in cases], check)
    for c, r, v, out in zip(cases, rets, checks, outs):
        assert r == c.verdict, c.name
        if c.verdict == 0:
            assert out == c.expected, c.name
            assert v == crc(check, c.expected), c.name


def test_stream_decode_sized_and_unsized(ctx, cases):
    for c in cases:
        for xz in (c.xz, X.drop_block_sizes(c.xz)):
            r, back = ctx.stream_decode(xz, c.declared)
            assert r == c.verdict, c.name
            if c.verdict == 0:
                assert back == c.expected, c.name


def dev_batch(ctx, streams, caps, flags=0):
    """xzb_stream_buffer_decode_batch_device with Streams and slots at odd offsets: [(ret, output, in_used)]."""
    in_off, in_total = _odd_offsets([len(s) for s in streams], 1)
    out_off, out_total = _odd_offsets(caps, 3)
    src = bytearray(in_total)
    for o, s in zip(in_off, streams):
        src[o:o + len(s)] = s
    d_in, d_out = ctx.device_alloc(in_total), ctx.device_alloc(out_total)
    try:
        ctx.h2d(d_in, bytes(src), in_total)
        res = ctx.stream_buffer_decode_batch_device(d_in, in_off, [len(s) for s in streams], d_out, out_off, caps, flags)
        back = bytearray(out_total)
        ctx.d2h(back, d_out, out_total)
    finally:
        ctx.device_free(d_in); ctx.device_free(d_out)
    return [(r, bytes(back[o:o + size]), used) for o, (r, size, used) in zip(out_off, res)]


def test_stream_batches(ctx, cases):
    """Every Stream, sized and unsized, in one host batch and one device batch.  Near misses: the verdict only."""
    items = [(c, xz) for c in cases for xz in (c.xz, X.drop_block_sizes(c.xz))]
    streams, caps = [xz for _, xz in items], [c.declared for c, _ in items]
    for got in (ctx.stream_buffer_decode_batch(streams, caps), dev_batch(ctx, streams, caps)):
        assert len(got) == len(items)
        for (c, xz), (r, out, used) in zip(items, got):
            if c.verdict == 0:
                assert (r, out, used) == (0, c.expected, len(xz)), c.name
            else:
                assert r == c.verdict, c.name


# ---- check kernels ----

def crc_sizes():
    """xzb_k_crc splits n bytes into a short leading slice of r bytes and k <= 1023 slices of L = ceil(n / 1023) bytes."""
    sizes = [0, 1, 2, 63, 64, 65] + list(range(1021, 1026)) + list(range(2045, 2049))
    for L in (2, 3, 64, 4097):
        sizes += [1023 * L - 1, 1023 * L, 1023 * L + 1]
    return sorted(set(sizes)) + [64 * MiB - 1, 64 * MiB, 64 * MiB + 1]


def test_crc_kernel_slicing_edges(ctx):
    """All sizes in one call, so the grid mixes them; payloads of uncompressed chunks only."""
    sizes = crc_sizes()
    datas = [G.filler(n, n) for n in sizes]
    payloads = [G.uncompressed_payload(d) for d in datas]
    for check in (1, 4):
        rets, checks, outs = decode_blocks(ctx, payloads, sizes, [1 << 26] * len(sizes), check)
        assert rets == [0] * len(sizes)
        for n, d, v, out in zip(sizes, datas, checks, outs):
            assert out == d, n
            assert v == crc(check, d), (check, n)


def check_streams():
    """(check, size, Stream) with CRC32, CRC64 and SHA-256 Check fields: every size 0..130 (SHA-256 pads at 55 / 56 /
    63 / 64 / 119 / 120 ...), 1 MiB and its neighbours, and some of the CRC kernel's slicing edges."""
    sizes = list(range(131)) + [MiB - 1, MiB, MiB + 1, 2045, 2046, 2047, 2048, 1023 * 64 - 1, 1023 * 64, 1023 * 64 + 1]
    out = []
    for check in (1, 4, 10):
        for n in sizes:
            d = G.filler(7 * n + check, n)
            out.append((check, d, G.xz_stream(G.uncompressed_payload(d), 0, n, check, d)))
    return out


def flip_check_bit(xz, k):
    """xz with bit k (mod the field's size) of its Check field flipped."""
    csize = {1: 4, 4: 8, 10: 32}[xz[7]]
    index_size = (struct.unpack_from("<I", xz, len(xz) - 8)[0] + 1) * 4
    at = len(xz) - 12 - index_size - csize + (k // 8) % csize
    bad = bytearray(xz)
    bad[at] ^= 1 << (k % 8)
    return bytes(bad)


def test_check_fields_through_stream_batches(ctx):
    items = check_streams()
    good = [xz for _, _, xz in items]
    bad = [flip_check_bit(xz, 13 * i) for i, xz in enumerate(good)]
    caps = [len(d) for _, d, _ in items]
    for decode in (ctx.stream_buffer_decode_batch, lambda s, c, f=0: dev_batch(ctx, s, c, f)):
        for streams, flags, want in ((good, 0, 0), (bad, 0, 9), (bad, IGNORE_CHECK, 0)):
            got = decode(streams, caps, flags)
            for (check, d, _), xz, (r, out, used) in zip(items, streams, got):
                assert r == want, (check, len(d), flags)
                if want == 0:
                    assert out == d and used == len(xz), (check, len(d))

