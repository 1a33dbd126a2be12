"""CPU tests of the resumable Block decoder (xz_b200/csrc/xzb_dec_resume.cuh, the body of xzb_block_decoder_*), run through
tests/hostsim/block_dec_host.cpp with the host form of the chunk decoder, CRC and SHA-256 in place of the kernels.

Every Block is decoded four ways -- input cut at every LZMA2 chunk boundary (one chunk per piece, and the smallest
window the decoder may keep), input cut at seeded random byte positions, output taken 1, 7 and 4096 bytes per call, and
all in one piece -- and must give the bytes and the verdict of the whole-Block decoder (tests/hostsim/dec_stream_host.cpp,
itself pinned to the reference's recorded verdicts):
  * every case of tests/lzma2_gen.py (mid-Block resets, new lc/lp/pb, window edges, near misses), sized and unsized;
    the window_* cases (4-8 KiB dictionaries, distances of full - 1 across mid-Block resets) slide the window many
    times.  The harness garbles every window byte older than min(bytes out, dict_size_r) before each piece, and the
    model when a piece's first chunk resets it (the kernel does not load it then), so the bytes only come out right if
    the decoder never needs more history than the dictionary and never a model it did not keep;
  * every Block of every case of tests/chunk_mix.py;
  * every LZMA2-only Block of the reference's decoder corpus (tests/golden/ref_files), the broken ones included."""
import ctypes as C
import functools
import os
import random
import struct
import zlib

import pytest

import chunk_mix as M
import lzma2_gen as G
import xzlibs as X

DATA_ERROR, BUF_ERROR, STREAM_END = 9, 10, 1


@pytest.fixture(scope="module")
def bd():
    lib = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libblockdechost.so"))
    lib.bd_run.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def ds():
    lib = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libdecstreamhost.so"))
    lib.ds_decode_batch.restype = C.c_int
    return lib


def whole(ds, xz, cap):
    """(ret, bytes) of the whole-Block decoder on one Stream (lzma_stream_buffer_decode's mapping)."""
    A = C.c_uint64 * 1
    src = (C.c_uint8 * max(len(xz), 1)).from_buffer_copy(xz or b"\0")
    out = (C.c_uint8 * max(cap, 1))()
    size, used, ret, rounds = A(), A(), (C.c_uint32 * 1)(), C.c_uint32()
    assert ds.ds_decode_batch(C.c_uint32(1), src, A(0), A(len(xz)), out, A(0), A(cap), size, used, ret, C.c_uint32(0), C.c_uint32(65536),
                              C.byref(rounds)) == 0
    return ret[0], bytes(out[: size[0]])


def run(bd, blk, check, cuts=(), out_step=0, piece_in=0, piece_out=0, cap=None):
    """(ret, bytes, in_used, stats, record) of the resumable decoder on one Block."""
    cap = cap if cap is not None else 64 << 20
    src = (C.c_uint8 * max(len(blk), 1)).from_buffer_copy(blk or b"\0")
    out = (C.c_uint8 * max(cap, 1))()
    cuts = sorted(set(cuts))
    cu = (C.c_uint64 * max(len(cuts), 1))(*cuts)
    osz, iu, stats, rec = C.c_uint64(), C.c_uint64(), (C.c_uint64 * 8)(), (C.c_uint64 * 2)()
    r = bd.bd_run(src, C.c_uint64(len(blk)), C.c_uint32(check), C.c_uint32(0), cu, C.c_uint32(len(cuts)), C.c_uint64(out_step),
                  C.c_uint64(piece_in), C.c_uint64(piece_out), out, C.c_uint64(cap), C.byref(osz), C.byref(iu), stats, rec)
    return r, bytes(out[: osz.value]), iu.value, list(stats), (rec[0], rec[1])


def header_size(blk):
    return (blk[0] + 1) * 4


def chunk_cuts(blk):
    """Offsets in the Block of every LZMA2 chunk boundary (as far as the chunk headers can be read)."""
    p, cuts = header_size(blk), []
    while p < len(blk):
        c = blk[p]
        cuts.append(p)
        if c == 0:
            break
        if c >= 0x80:
            if p + 5 > len(blk):
                break
            p += (6 if c >= 0xC0 else 5) + (blk[p + 3] << 8) + blk[p + 4] + 1
        elif c <= 2:
            if p + 3 > len(blk):
                break
            p += 3 + (blk[p + 1] << 8) + blk[p + 2] + 1
        else:
            break
    return cuts


def blocks(xz, measure=None):
    """(Block bytes, check) of every Block of the first Stream: sized Blocks end where their headers say; an unsized
    Block ends where measure(rest of the input, check) -- the bytes a decoder consumed -- says, and without `measure`
    (or when measure gives 0) it takes the rest of the input and ends the list."""
    check = xz[7] & 0x0F
    csize = 0 if check == 0 else 4 << ((check - 1) // 3)
    p, out = 12, []
    while p < len(xz) and xz[p] != 0:
        hs = (xz[p] + 1) * 4
        flags = xz[p + 1]
        if p + hs > len(xz):
            break
        if flags & 0x40:
            comp, _ = X._read_vli(xz, p + 2)
            end = p + hs + ((comp + 3) & ~3) + csize
            out.append((xz[p:end], check))
            p = end
        else:
            n = measure(xz[p:], check) if measure else 0
            if n <= hs:
                out.append((xz[p:], check))
                break
            out.append((xz[p:p + n], check))
            p += n
    return out


def _ended(res):
    """The bytes a decode result consumed when its Block ended, else 0."""
    return res[2] if res[0] == STREAM_END else 0


def _first_filter(blk):
    q = 2
    for bit in (0x40, 0x80):
        if blk[1] & bit:
            _, q = X._read_vli(blk, q)
    fid, _ = X._read_vli(blk, q)
    return fid


def four_ways(bd, blk, check, seed, cap):
    """The cut patterns; yields (label, result)."""
    cuts = chunk_cuts(blk)
    yield "chunks", run(bd, blk, check, cuts=cuts, piece_in=1, piece_out=1, cap=cap)
    rnd = random.Random(seed)
    yield "random", run(bd, blk, check, cuts=[rnd.randrange(len(blk) + 1) for _ in range(24)], cap=cap)
    for step in (1, 7, 4096):
        yield "out%d" % step, run(bd, blk, check, out_step=step, cap=cap)
    yield "one", run(bd, blk, check, cap=cap)


def same(label, got, want_ret, want_out, name):
    r, out = got[0], got[1]
    assert out == want_out[: len(out)], (name, label, "bytes differ")
    if want_ret == 0:
        assert r == STREAM_END and out == want_out, (name, label, r)
    else:
        assert r == want_ret and out == want_out, (name, label, r, want_ret, len(out), len(want_out))


GEN = G.cases()


@pytest.mark.parametrize("case", GEN, ids=[c.name for c in GEN])
def test_lzma2_gen_cases_in_pieces(bd, ds, case):
    for form, xz in (("sized", case.xz), ("unsized", X.drop_block_sizes(case.xz))):
        (blk, check), = blocks(xz)
        want_ret, want_out = whole(ds, xz, max(case.declared, 1) + 4096)
        assert want_ret == case.verdict
        if case.verdict == 0:
            assert want_out == case.expected
        for label, got in four_ways(bd, blk, check, sum(case.name.encode()), len(want_out) + 4096):
            same(label, got, want_ret, want_out, (case.name, form))
            if got[0] == STREAM_END:
                hs = header_size(blk)
                csize = 0 if check == 0 else 4 << ((check - 1) // 3)
                assert got[4] == (hs + len(case.payload) + csize, len(case.expected))
                assert got[2] == hs + ((len(case.payload) + 3) & ~3) + csize


def test_window_cases_slide_the_window(bd):
    """The small-dictionary cases fed a chunk at a time really move their history to the front."""
    wins = [c for c in GEN if c.name.startswith("window_")]
    assert wins
    for c in wins:
        (blk, check), = blocks(c.xz)
        r, out, _, st, _ = run(bd, blk, check, cuts=chunk_cuts(blk), piece_in=1, piece_out=1, cap=len(c.expected) + 4096)
        assert r == STREAM_END and out == c.expected
        assert st[1] >= 1 and 0 < st[3] <= st[4], (c.name, st)   # slides, each moving at most a dictionary


@functools.lru_cache(maxsize=1)
def _mix_streams():
    return [(c.name, M.oracle_counters(c)[0], c.data) for c in M.cases()]


@pytest.mark.parametrize("i", range(len(M.cases())))
def test_chunk_mix_blocks_in_pieces(bd, ds, i):
    name, xz, data = _mix_streams()[i]
    pos = 0
    for k, (blk, check) in enumerate(blocks(xz)):
        res = list(four_ways(bd, blk, check, 1000 * i + k, len(data) + 4096))
        r0, out0 = res[-1][1][0], res[-1][1][1]
        assert r0 == STREAM_END
        assert out0 == data[pos: pos + len(out0)], (name, k)
        for label, got in res:
            same(label, got, 0, out0, (name, k))
        pos += len(out0)
    assert pos == len(data)


def _corpus():
    d = os.path.join(X.ROOT, "tests", "golden", "ref_files")
    out = []
    lib = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libblockdechost.so"))
    lib.bd_run.restype = C.c_int
    measure = lambda b, c: _ended(run(lib, b, c, cap=1 << 20))
    for n in sorted(os.listdir(d)):
        xz = open(os.path.join(d, n), "rb").read()
        if len(xz) < 12 or xz[:6] != b"\xfd7zXZ\x00":
            continue
        for k, (blk, check) in enumerate(blocks(xz, measure)):
            try:
                if _first_filter(blk) == 0x21 and (blk[1] & 3) == 0:
                    out.append((n, k, blk, check, xz))
            except IndexError:
                pass
    return out


CORPUS = _corpus()


@pytest.mark.parametrize("item", CORPUS, ids=["%s#%d" % (c[0], c[1]) for c in CORPUS])
def test_reference_corpus_blocks_in_pieces(bd, ds, item):
    """A corpus Block gives the whole-Block decoder's bytes; where the resumable decoder fails, the whole file fails with
    the same verdict (input that ends early inside the Block is LZMA_BUF_ERROR for a streaming caller, LZMA_DATA_ERROR
    under the one-shot mapping)."""
    name, k, blk, check, xz = item
    # (under a valid Stream Header with the file's Check ID: a broken one ends the whole-Stream decode before any Block)
    flags = bytes([0, check])
    want_ret, want_out = whole(ds, b"\xfd7zXZ\x00" + flags + struct.pack("<I", zlib.crc32(flags)) + xz[12:], 1 << 20)
    measure = lambda b, c: _ended(run(bd, b, c, cap=1 << 20))
    base = len(b"".join(run(bd, b, c, cap=1 << 20)[1] for b, c in blocks(xz, measure)[:k]))
    for label, got in four_ways(bd, blk, check, k, 1 << 20):
        r, out = got[0], got[1]
        assert out == want_out[base: base + len(out)], (name, k, label)
        if r != STREAM_END:
            assert (DATA_ERROR if r == BUF_ERROR else r) == want_ret, (name, k, label, r, want_ret)
            assert base + len(out) == len(want_out), (name, k, label)
