"""GPU tests of lzma_stream_decoder[_mt] + lzma_code on Blocks decoded piece by piece (xzb_block_decoder_*):
  (b) single-Block Streams without sizes (X.drop_block_sizes of oracle Streams, -1 / -6, all four checks), fed 8 KiB or
      1 MiB at a time under LZMA_RUN or LZMA_FINISH: the bytes are right and output appears before the last third of
      the input is fed; a flipped byte in the last chunk, a wrong Check field and a truncated Stream give the earlier
      bytes and then LZMA_DATA_ERROR / LZMA_DATA_ERROR / LZMA_BUF_ERROR;
  (c) more than 4 GiB in one Block (the synthetic Block of test_gpu_block_decoder.py), unsized and sized, streamed
      through lzma_code into a 64 MiB buffer in bounded memory;
  (d) sized Blocks, an unsized one, sized ones, Stream Padding and a second Stream under LZMA_CONCATENATED, and a wrong
      Index record of the unsized Block caught at the Index;
  (e) LZMA_MEMLIMIT_ERROR before the unsized Block's first byte, and lzma_memlimit_set() recovers."""
import ctypes as C
import resource
import struct

import pytest

import test_gpu_block_decoder as TB
import xz_b200
import xzlibs as X
from test_api_cpu import LzmaMt, LzmaStream

pytestmark = pytest.mark.gpu
RUN, FINISH = 0, 3


@pytest.fixture(scope="module")
def lib():
    L = xz_b200.lib()
    L.lzma_memusage.restype = C.c_uint64
    return L


def decoder(lib, mt=False, flags=0, memlimit=(1 << 64) - 1):
    s = LzmaStream()
    if mt:
        m = LzmaMt(); m.flags = flags; m.threads = 4; m.memlimit_stop = memlimit; m.memlimit_threading = memlimit
        assert lib.lzma_stream_decoder_mt(C.byref(s), C.byref(m)) == 0
    else:
        assert lib.lzma_stream_decoder(C.byref(s), C.c_uint64(memlimit), C.c_uint32(flags)) == 0
    return s


def drive(lib, s, stream, step, final=FINISH, sink=None, out_cap=1 << 16):
    """Feed `stream` `step` bytes at a time (the last call with `final`); returns (ret, output, input fed when the first
    output appeared).  sink(chunk) takes the output instead when given."""
    ibuf = (C.c_uint8 * max(len(stream), 1)).from_buffer_copy(stream or b"\0")
    obuf = (C.c_uint8 * out_cap)()
    out, pos, first, ret = bytearray(), 0, None, 0
    s.next_out, s.avail_out = C.addressof(obuf), out_cap
    for _ in range(10_000_000):
        if s.avail_in == 0 and pos < len(stream):
            k = min(step, len(stream) - pos)
            s.next_in, s.avail_in = C.addressof(ibuf) + pos, k
            pos += k
        ret = lib.lzma_code(C.byref(s), final if pos == len(stream) else RUN)
        got = out_cap - s.avail_out
        if got:
            if first is None:
                first = pos
            if sink:
                sink(C.string_at(obuf, got))
            else:
                out += C.string_at(obuf, got)
            s.next_out, s.avail_out = C.addressof(obuf), out_cap
        if ret != 0:
            break
    lib.lzma_end(C.byref(s))
    return ret, bytes(out), first


def one_block(kind, n, preset, check):
    buf = X.gendata(kind, n)
    return bytes(buf[:n]), X.drop_block_sizes(X.oracle_encode(buf, n, preset, n, check))


@pytest.mark.parametrize("preset,check", [(1, 1), (6, 4), (1, 10), (6, 0)], ids=["p1-crc32", "p6-crc64", "p1-sha256", "p6-none"])
def test_unsized_stream_through_lzma_code(lib, preset, check):
    data, xz = one_block("E", 12 << 20, preset, check)
    assert len(xz) > (3 << 20)   # several pieces of input, also in 1 MiB feeds
    for mt, step, final in ((False, 8192, FINISH), (True, 8192, RUN), (False, 1 << 20, RUN), (True, 1 << 20, FINISH)):
        ret, out, first = drive(lib, decoder(lib, mt), xz, step, final)
        assert ret == 1 and out == data, (mt, step, final, ret)
        assert first is not None and first < len(xz) * 2 // 3, (mt, step, final, first, len(xz))


def test_unsized_stream_corruptions(lib):
    data, xz = one_block("E", 6 << 20, 1, 1)
    idx = (int.from_bytes(xz[-8:-4], "little") + 1) * 4
    block_end = len(xz) - 12 - idx               # after the Check field
    # a flipped byte in the last chunk: the earlier bytes, then LZMA_DATA_ERROR
    bad = bytearray(xz); bad[block_end - 4 - 3 - 60] ^= 0x10
    ret, out, _ = drive(lib, decoder(lib), bytes(bad), 8192)
    keep = len(data) - (2 << 20)   # everything before the last chunk
    assert ret == 9 and len(out) >= keep and out[:keep] == data[:keep]
    # a wrong Check field: every byte, then LZMA_DATA_ERROR
    bad = bytearray(xz); bad[block_end - 1] ^= 0x01
    ret, out, _ = drive(lib, decoder(lib), bytes(bad), 8192)
    assert ret == 9 and out == data
    # a truncated Stream: LZMA_OK with what was decodable, then LZMA_BUF_ERROR on the next call without progress
    ret, out, _ = drive(lib, decoder(lib), xz[: len(xz) // 2], 8192)
    assert ret == 10 and out == data[: len(out)] and len(out) > 0


def _records(xz):
    back = (struct.unpack_from("<I", xz, len(xz) - 8)[0] + 1) * 4
    count, p = X._read_vli(xz, len(xz) - 12 - back + 1)
    recs = []
    for _ in range(count):
        u, p = X._read_vli(xz, p)
        v, p = X._read_vli(xz, p)
        recs.append((u, v))
    return recs


def mixed_stream(buf, n, bs, check, unsized_at, bump=0):
    """The oracle's Stream of n bytes in bs Blocks with Block `unsized_at` written without sizes; bump is added to that
    Block's Uncompressed Size in the Index (a wrong record)."""
    a = X.oracle_encode(buf, n, 1, bs, check)
    u = X.drop_block_sizes(a)
    ra, ru = _records(a), _records(u)
    body, recs, pa, pu = bytearray(), [], 12, 12
    for i in range(len(ra)):
        la, lu = (ra[i][0] + 3) & ~3, (ru[i][0] + 3) & ~3
        if i == unsized_at:
            body += u[pu: pu + lu]; recs.append((ru[i][0], ru[i][1] + bump))
        else:
            body += a[pa: pa + la]; recs.append(ra[i])
        pa += la; pu += lu
    idx = xz_b200.index_encode(recs)
    return a[:12] + bytes(body) + idx + xz_b200.stream_footer(check, len(idx))


def test_mixed_stream_concatenated(lib):
    n, bs = 5 << 20, 1 << 20
    buf = X.gendata("T", n)
    data = bytes(buf[:n])
    one = mixed_stream(buf, n, bs, 4, 2)
    two = mixed_stream(buf, n, bs, 10, 0)
    for step in (8192, 1 << 20):
        ret, out, _ = drive(lib, decoder(lib, flags=0x08), one + bytes(8) + two, step)
        assert ret == 1 and out == data + data, step
    bad = mixed_stream(buf, n, bs, 4, 2, bump=1)
    ret, out, _ = drive(lib, decoder(lib), bad, 8192)
    assert ret == 9 and out == data


def test_memlimit_before_the_unsized_block(lib):
    data, xz = one_block("T", 1 << 20, 6, 4)        # -6: an 8 MiB dictionary
    s = decoder(lib, memlimit=1 << 20)
    ibuf = (C.c_uint8 * len(xz)).from_buffer_copy(xz)
    obuf = (C.c_uint8 * (2 << 20))()
    s.next_in, s.avail_in, s.next_out, s.avail_out = C.addressof(ibuf), len(xz), C.addressof(obuf), len(obuf)
    assert lib.lzma_code(C.byref(s), FINISH) == 6     # LZMA_MEMLIMIT_ERROR
    assert s.total_out == 0
    need = lib.lzma_memusage(C.byref(s))
    assert need == (8 << 20) + 66200
    assert lib.lzma_memlimit_set(C.byref(s), C.c_uint64(need - 1)) == 6
    assert lib.lzma_memlimit_set(C.byref(s), C.c_uint64(need)) == 0
    ret = 0
    for _ in range(100):
        ret = lib.lzma_code(C.byref(s), FINISH)
        if ret != 0:
            break
    assert ret == 1 and bytes(obuf[: s.total_out]) == data
    lib.lzma_end(C.byref(s))


@pytest.mark.parametrize("sized", [False, True], ids=["unsized", "sized"])
@pytest.mark.parametrize("check,reps", [(1, 2560), (10, 128)], ids=["crc32-5GiB", "sha256-256MiB"])
def test_block_over_4gib_through_lzma_code(lib, sized, check, reps):
    payload, headb, fill, total = TB.synthetic(reps)
    cf = TB.expected_check(headb, fill, total, check)
    blk = TB.block_bytes(payload, total, check, cf, sized)
    idx = xz_b200.index_encode([(len(blk) - (-len(payload) % 4), total)])
    xz = xz_b200.stream_header(check) + blk + idx + xz_b200.stream_footer(check, len(idx))
    fill_run = bytes([fill]) * (64 << 20)
    got = [0]

    def sink(chunk):
        g, k = got[0], 0
        if g < 64:
            k = min(64 - g, len(chunk))
            assert chunk[:k] == headb[g: g + k]
        assert chunk[k:] == fill_run[: len(chunk) - k]
        got[0] += len(chunk)

    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    ret, _, first = drive(lib, decoder(lib), xz, 1 << 20, sink=sink, out_cap=64 << 20)
    rss1 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    assert ret == 1 and got[0] == total
    assert (rss1 - rss0) * 1024 < (1 << 30), (rss0, rss1)
