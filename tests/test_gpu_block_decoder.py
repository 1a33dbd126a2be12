"""GPU tests of the resumable Block decoder (xzb_block_decoder_*, kernel xzb_k_decode_resume):
  (a) the C ABI against the whole-Block kernel: Blocks of tests/lzma2_gen.py (sized and unsized), of oracle-encoded
      Streams and of the reference's corpus, fed cut at every chunk boundary, at seeded random byte positions, with small
      output buffers and in one piece, give the bytes and the verdict xzb_stream_buffer_decode gives for their Streams;
  (c) more than 4 GiB in one Block, unsized and sized: a 0xE0 chunk and then one 0xA0 chunk of rep0 length-273
      matches, repeated (its unpacked size is a multiple of 4, so with lp = 0 and pb = 2 every copy codes the same),
      about 5 GiB of output from a few MB of input, handed out through a 64 MiB buffer and hashed on the fly: the bytes
      and the CRC32 check are right and the process's peak RSS grows by less than 1 GiB.  The same Stream with a
      SHA-256 check at 256 MiB of output."""
import hashlib
import os
import random
import resource
import struct
import zlib

import pytest

import lzma2_gen as G
import xz_b200
import xzlibs as X
from test_block_decoder_cpu import _ended, blocks, chunk_cuts, header_size

pytestmark = pytest.mark.gpu
STREAM_END, DATA_ERROR, BUF_ERROR = 1, 9, 10


@pytest.fixture(scope="module")
def ctx():
    c = xz_b200.Context(0)
    yield c
    c.close()


def feed(ctx, blk, check, cuts=(), out_cap=1 << 20):
    """(ret, bytes, in_used) of xzb_block_decoder over one Block, the input growing through `cuts`."""
    hs = header_size(blk)
    bd = ctx.block_decoder(blk[:hs], check)
    pos, have, out = hs, None, bytearray()
    cuts = sorted(c for c in set(cuts) if c > hs) + [len(blk)]
    k = 0
    have = cuts[0]
    for _ in range(10_000_000):
        r, o, used = bd.code(blk[pos:have], out_cap, have == len(blk))
        out += o
        pos += used
        if r != 0:
            break
        if not o and not used:
            assert have < len(blk), "no progress with all input in"
            k += 1
            have = cuts[k]
    rec = bd.record() if r == STREAM_END else None
    bd.close()
    return r, bytes(out), pos, rec


def patterns(blk, n_out, seed):
    yield "chunks", dict(cuts=chunk_cuts(blk))
    rnd = random.Random(seed)
    yield "random", dict(cuts=[rnd.randrange(len(blk) + 1) for _ in range(16)])
    for cap in (1, 7, 4096):
        if n_out // cap <= 20000:
            yield "out%d" % cap, dict(out_cap=cap)
    yield "one", dict(out_cap=max(n_out, 1))


def streams():
    out = []
    for c in G.cases():
        if c.declared <= 4 << 20:
            out.append((c.name, c.xz))
            out.append((c.name + "-unsized", X.drop_block_sizes(c.xz)))
    for kind, preset, check in (("T", 1, X.CHECK_CRC32), ("E", 6, X.CHECK_CRC64), ("R", 1, 10), ("T", 6, 0)):
        buf = X.gendata(kind, 300000)
        xz = X.oracle_encode(buf, 300000, preset, 1 << 17, check)
        out.append(("%s%d-c%d" % (kind, preset, check), xz))
        out.append(("%s%d-c%d-unsized" % (kind, preset, check), X.drop_block_sizes(xz)))
    d = os.path.join(X.ROOT, "tests", "golden", "ref_files")
    for n in sorted(os.listdir(d)):
        if "lzma2" in n or "check" in n:
            out.append((n, open(os.path.join(d, n), "rb").read()))
    return out


STREAMS = streams()


@pytest.mark.parametrize("name,xz", STREAMS, ids=[s[0] for s in STREAMS])
def test_block_decoder_matches_whole_block_kernel(ctx, name, xz):
    want_ret, want, _ = ctx.stream_buffer_decode(xz, 8 << 20)
    done = 0
    for k, (blk, check) in enumerate(blocks(xz, lambda b, c: 0 if b[1] & 3 else _ended(feed(ctx, b, c)))):
        if (blk[1] & 3) != 0:   # a Delta / BCJ chain in front of LZMA2 is not for this decoder
            with pytest.raises(xz_b200.XzError) as e:
                ctx.block_decoder(blk[:header_size(blk)], check)
            assert e.value.code == 8   # LZMA_OPTIONS_ERROR
            return
        for label, kw in patterns(blk, len(want) - done, k):
            r, out, _, _ = feed(ctx, blk, check, **kw)
            assert out == want[done: done + len(out)], (name, k, label)
            if r != STREAM_END:
                assert (DATA_ERROR if r == BUF_ERROR else r) == want_ret and done + len(out) == len(want), (name, k, label, r, want_ret)
        r, out, _, _ = feed(ctx, blk, check)
        if r != STREAM_END:
            return
        done += len(out)
    if want_ret == 0:
        assert done == len(want)


# ---- (c) more than 4 GiB in one Block ----
COPY = 273 * 7680       # unpacked bytes of one 0xA0 chunk


def synthetic(reps):
    """(Block, pattern head, byte repeated, total output) of the high-ratio Block."""
    b = G.Block(77, 18, G.Coverage())    # 2 MiB dictionary

    def head(bb, rc):
        for i in range(64):
            bb.literal(rc, 0x41 + (i % 26))
        return None

    def body(bb, rc):
        for _ in range(7680):
            bb.rep(rc, 0, 273)
        return None

    b.lzma(0xE0, 64, None, (3, 0, 2), script=head)
    first = len(b.payload)
    b.lzma(0xA0, COPY, None, script=body)
    chunk = bytes(b.payload[first:])
    payload = bytes(b.payload[:first]) + chunk * reps + b"\x00"
    total = 64 + COPY * reps
    headb, fill = bytes(b.out[:64]), b.out[63]
    return payload, headb, fill, total


def block_bytes(payload, total, check, cfield, sized):
    flags = 0xC0 if sized else 0x00
    body = bytes([flags]) + ((G._vli(len(payload)) + G._vli(total)) if sized else b"") + b"\x21\x01" + bytes([18])
    body += b"\0" * (-(len(body) + 5) % 4)
    hdr = bytes([(len(body) + 5) // 4 - 1]) + body
    hdr += struct.pack("<I", zlib.crc32(hdr))
    return hdr + payload + b"\0" * (-len(payload) % 4) + cfield


def expected_check(headb, fill, total, check):
    run = bytes([fill]) * (64 << 20)
    h = hashlib.sha256(headb) if check == 10 else None
    c = zlib.crc32(headb)
    left = total - len(headb)
    while left:
        k = min(left, len(run))
        if h:
            h.update(run[:k])
        else:
            c = zlib.crc32(run[:k], c)
        left -= k
    return h.digest() if h else struct.pack("<I", c)


@pytest.mark.parametrize("sized", [False, True], ids=["unsized", "sized"])
@pytest.mark.parametrize("check,reps", [(1, 2560), (10, 128)], ids=["crc32-5GiB", "sha256-256MiB"])
def test_block_over_4gib_in_bounded_memory(ctx, sized, check, reps):
    import ctypes as C
    payload, headb, fill, total = synthetic(reps)
    cfield = expected_check(headb, fill, total, check)
    blk = block_bytes(payload, total, check, cfield, sized)
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    hs = header_size(blk)
    bd = ctx.block_decoder(blk[:hs], check)
    cap = 64 << 20
    obuf = (C.c_uint8 * cap)()
    src = (C.c_uint8 * len(blk)).from_buffer_copy(blk)
    fill_run = bytes([fill]) * cap
    pos, got, r = hs, 0, 0
    while True:
        r, n, used = bd.code_into(C.addressof(src) + pos, len(blk) - pos, obuf, cap, True)
        pos += used
        if n:
            view = bytes(obuf[:n]) if got < 64 else None
            if got < 64:
                k = min(64 - got, n)
                assert view[:k] == headb[got: got + k]
                assert view[k:] == fill_run[: n - k]
            else:
                assert C.string_at(obuf, n) == fill_run[:n]
            got += n
        if r != 0:
            break
    st = bd.stats()
    rec = bd.record() if r == STREAM_END else None
    bd.close()
    rss1 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    assert r == STREAM_END and got == total and pos == len(blk)
    assert rec == (hs + len(payload) + len(cfield), total)
    assert (rss1 - rss0) * 1024 < (1 << 30), (rss0, rss1)
    assert st.window_bytes < (1 << 30) and st.pieces > 1
    print("\n%s %s: %d bytes, %d pieces, %d slides (%d B), window %d B, decode %.1f ms, check %.1f ms, d2h %.1f ms"
          % ("sized" if sized else "unsized", check, got, st.pieces, st.slides, st.bytes_slid, st.window_bytes, st.ms_decode, st.ms_check,
             st.ms_d2h))
