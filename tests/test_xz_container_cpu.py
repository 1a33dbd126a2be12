"""CPU tests of the .xz container read side (xz_b200/csrc/xzb_frame.cuh), compiled into tests/hostsim: the Stream
Header / Footer, Block Header (framing only and full parse) and Index readers that the decoder and the liblzma-named
stream coders of libxzb200.so walk a Stream with.
  * Streams from the oracle: the Block walk yields the records written into the Index, no strict prefix is complete,
    the whole Stream is, and the Index check accepts the Stream's own records and rejects a changed one;
  * the corpus of tests/golden/ref_files and the generated trace inputs, every prefix and every single-byte flip:
    every reader answers from inside the buffer it was given."""
import ctypes as C
import os
import sys

import pytest

import xzlibs as X

GOLD = os.path.join(X.ROOT, "tests", "golden")
OK, DATA_ERROR = 0, 9
VLI_LONG = 2
N = 20000  # uncompressed bytes of each oracle Stream


class IndexRecord(C.Structure):
    _fields_ = [("unpadded_size", C.c_uint64), ("uncompressed_size", C.c_uint64)]


@pytest.fixture(scope="module")
def hs():
    return C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libhostsim.so"))


def _index_read(hs, buf, at, size, want=None):
    """(verdict, count, listed, end, stop) of the Index at buf[at .. size)."""
    o = (C.c_uint64 * 4)()
    w = (IndexRecord * max(len(want), 1))(*want) if want is not None else None
    r = hs.hs_index_read(C.byref(buf, at), C.c_uint64(size - at), w, C.c_uint64(len(want) if want is not None else 0), o)
    count, listed, end, stop = o
    assert r != OK or (listed and stop == end <= size - at)
    assert r == OK or stop <= size - at
    return r, count, bool(listed), end, stop


def walk(hs, buf, size):
    """The Stream at buf[0 .. size) through every reader: Stream Header; at each Block the framing read and the full
    parse; the sized Blocks walked by their framing to the Index; the Index and the Stream Footer behind it.
    Returns (complete, end, Check ID of a valid Stream Header or None, records of the Block walk, Index verdict)."""
    if size < 12:
        return False, 0, None, [], None
    chk = C.c_uint32()
    check = chk.value if hs.hs_stream_header_decode(buf, C.byref(chk)) == OK else None
    c = buf[7] & 0x0F
    csize = 0 if c == 0 else 4 << ((c - 1) // 3)
    ip, recs = 12, []
    while True:
        if ip >= size:
            return False, 0, check, recs, None
        if buf[ip] == 0:
            break
        hb = (C.c_uint64 * 11)()
        r = hs.hs_block_header_decode(C.byref(buf, ip), C.c_uint64(size - ip), hb)
        o = (C.c_uint64 * 8)()
        if not hs.hs_block_framing(C.byref(buf, ip), C.c_uint64(size - ip), o):
            assert r != OK
            return False, 0, check, recs, None
        hsize, flags, comp, comp_end, comp_st, uncomp, uncomp_end, _ = o
        assert comp_end <= hsize and uncomp_end <= hsize <= size - ip
        if r == OK:
            assert hb[0] == hsize and hb[4] <= 3 and (hb[1] == comp or not flags & 0x40)
        if not flags & 0x40 or comp_st == VLI_LONG:
            return False, 0, check, recs, None
        total = hsize + ((comp + 3) & ~3) + csize
        if size - ip < total:
            return False, 0, check, recs, None
        recs.append((hsize + comp + csize, uncomp))
        ip += total
    r, _, listed, end, _ = _index_read(hs, buf, ip, size, recs)
    if not listed or size - ip < end + 12:
        return False, 0, check, recs, r
    fchk, isize = C.c_uint32(), C.c_uint64()
    if hs.hs_stream_footer_decode(C.byref(buf, ip + end), C.byref(fchk), C.byref(isize)) == OK:
        assert fchk.value <= 15 and isize.value % 4 == 0
    return True, ip + end + 12, check, recs, r


def _oracle_streams():
    buf = X.gendata("T", N)
    for check in (0, 1, 4, 10):
        for bs in (N, 7000, 3000):
            yield f"check{check}-bs{bs}", X.oracle_encode(buf, N, 1, bs, check=check), check, -(-N // bs)
        yield f"check{check}-oneshot", X.oracle_buffer_encode(buf, N, 1, check=check), check, 1


@pytest.mark.parametrize("name,xz,check,nblocks", list(_oracle_streams()), ids=lambda v: v if isinstance(v, str) and len(v) < 40 else "")
def test_oracle_stream_walks_to_its_own_index(hs, name, xz, check, nblocks):
    n = len(xz)
    buf = (C.c_uint8 * n).from_buffer_copy(xz)
    complete, end, got_check, recs, verdict = walk(hs, buf, n)
    assert (complete, end, got_check, verdict, len(recs)) == (True, n, check, OK, nblocks)
    assert sum(u for _, u in recs) == N
    fchk, isize = C.c_uint32(), C.c_uint64()
    assert hs.hs_stream_footer_decode(C.byref(buf, n - 12), C.byref(fchk), C.byref(isize)) == OK and fchk.value == check
    at = n - 12 - isize.value
    assert _index_read(hs, buf, at, n - 12, recs)[:2] == (OK, nblocks)
    assert _index_read(hs, buf, at, n - 12, recs[:-1])[0] == DATA_ERROR
    for i in range(nblocks):
        for du, dc in ((1, 0), (0, 1)):
            bad = list(recs)
            bad[i] = (recs[i][0] + du, recs[i][1] + dc)
            assert _index_read(hs, buf, at, n - 12, bad)[0] == DATA_ERROR, (i, du, dc)
    for k in range(n):
        assert not walk(hs, buf, k)[0], k


def _corpus():
    sys.path.insert(0, GOLD)
    import make_golden as MG
    files = sorted(os.listdir(os.path.join(GOLD, "ref_files")))
    inputs = [(f, open(os.path.join(GOLD, "ref_files", f), "rb").read()) for f in files]
    return inputs + sorted(MG.trace_inputs().items())


def test_readers_stay_inside_every_prefix_and_flipped_byte(hs):
    for name, data in _corpus():
        n = len(data)
        buf = (C.c_uint8 * n).from_buffer_copy(data)
        for k in range(n + 1):
            complete, end = walk(hs, buf, k)[:2]
            assert not complete or end <= k, (name, k)
        for i in range(n):
            buf[i] ^= 0xFF
            complete, end = walk(hs, buf, n)[:2]
            assert not complete or end <= n, (name, i)
            if n > 12:  # the last 12 bytes as a Stream Footer, and the Index read from just behind the Stream Header
                fchk, isize = C.c_uint32(), C.c_uint64()
                hs.hs_stream_footer_decode(C.byref(buf, n - 12), C.byref(fchk), C.byref(isize))
                _index_read(hs, buf, 12, n)
            buf[i] ^= 0xFF
