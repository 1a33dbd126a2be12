"""CPU tests of the batch one-shot encoder's host pieces, compiled by tests/hostsim/batch_host.cpp: the wave planner and layout
(xz_b200/csrc/xzb_params.h) and the Stream framing that xzb_k_pack_streams runs (xz_b200/csrc/xzb_frame.cuh).
  * every item is placed exactly once, largest first; each wave keeps to the memory budget, the sort-key cap
    (B << hash_bits) < 2^32, sum(n) < 2^32 - 16 and the Block cap; every Block starts at a multiple of 256 positions;
  * the Block of an oracle one-shot Stream, framed again, is that Stream byte for byte."""
import ctypes as C
import os
import random
import struct

import pytest

import xzlibs as X

ALIGN = 256
GiB = 1 << 30


@pytest.fixture(scope="module")
def hs():
    lib = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libbatchhost.so"))
    lib.bh_plan_waves.restype = C.c_uint32
    lib.bh_pack_stream.restype = C.c_uint64
    return lib


def plan(hs, sizes, per_byte, per_block, budget, hash_bits, max_blocks=0):
    n = len(sizes)
    A = C.c_uint32 * max(n, 1)
    order, wave, off = A(), A(), A()
    nw = hs.bh_plan_waves((C.c_uint64 * max(n, 1))(*sizes), C.c_uint32(n), C.c_uint64(per_byte), C.c_uint64(per_block),
                          C.c_uint64(budget), C.c_uint32(hash_bits), C.c_uint32(max_blocks), order, wave, off)
    waves = [[] for _ in range(nw)]
    for k in range(n):
        waves[wave[k]].append((order[k], off[k]))
    return waves


def pad(v):
    return (v + ALIGN - 1) // ALIGN * ALIGN


def check_plan(sizes, waves, per_byte, per_block, budget, hash_bits, max_blocks=0):
    placed = [i for w in waves for i, _ in w]
    assert sorted(placed) == list(range(len(sizes)))
    assert [sizes[i] for i in placed] == sorted(sizes, reverse=True)  # largest first, across and within waves
    assert placed == sorted(placed, key=lambda i: (-sizes[i], i))      # ties keep the call order
    for w in waves:
        assert w, "empty wave"
        B, total = len(w), sum(pad(sizes[i]) for i, _ in w)
        assert B << hash_bits < 1 << 32 and total < (1 << 32) - 16
        assert max_blocks == 0 or B <= max_blocks
        assert B == 1 or per_byte * total + per_block * B <= budget
        pos = 0
        for i, off in w:
            assert off % ALIGN == 0 and off == pos
            pos += pad(sizes[i])


def test_planner_mixed_sizes_keep_every_limit(hs):
    rng = random.Random(7)
    sizes = [rng.choice((1, 255, 256, 257, 4096, 65537, 131072, 1 << 20, 3 << 20, 16 << 20)) + rng.randrange(64) for _ in range(1500)]
    for per_byte, per_block, budget, hash_bits, max_blocks in ((130, 75000, 60 << 30, 22, 0), (130, 75000, 2 << 30, 19, 0),
                                                              (100, 75000, 60 << 30, 19, 7), (200, 1 << 20, 1 << 28, 16, 0)):
        waves = plan(hs, sizes, per_byte, per_block, budget, hash_bits, max_blocks)
        check_plan(sizes, waves, per_byte, per_block, budget, hash_bits, max_blocks)
        if max_blocks:
            assert all(len(w) == max_blocks for w in waves[:-1])


@pytest.mark.parametrize("hash_bits,cap", [(22, 1023), (19, 8191)])
def test_planner_caps_blocks_by_sort_key_bits(hs, hash_bits, cap):
    """-6 (8 MiB dictionary, 22-bit hash): 1023 Blocks per wave; -1 (19-bit hash): 8191."""
    sizes = [4096] * 20000
    waves = plan(hs, sizes, 1, 0, 1 << 62, hash_bits)
    check_plan(sizes, waves, 1, 0, 1 << 62, hash_bits)
    assert [len(w) for w in waves[:-1]] == [cap] * (len(waves) - 1) and len(waves[-1]) <= cap


def test_planner_caps_positions_below_4_gib(hs):
    sizes = [GiB] * 7 + [GiB - 100, 5, 1]
    waves = plan(hs, sizes, 1, 0, 1 << 62, 16)
    check_plan(sizes, waves, 1, 0, 1 << 62, 16)
    assert [len(w) for w in waves] == [3, 3, 4]


def test_planner_oversized_item_runs_alone(hs):
    sizes = [1000, 50 << 20, 2000]
    waves = plan(hs, sizes, 100, 1000, 1 << 20, 16)
    check_plan(sizes, waves, 100, 1000, 1 << 20, 16)
    assert [i for i, _ in waves[0]] == [1]


def test_planner_no_items(hs):
    assert plan(hs, [], 100, 1000, 1 << 30, 22) == []


def _oneshot_block(xz):
    """(Block bytes, Unpadded Size, Uncompressed Size) of a one-Block Stream; (b"", 0, 0) for the Stream with no Block."""
    isize = (struct.unpack_from("<I", xz, len(xz) - 8)[0] + 1) * 4
    at = len(xz) - 12 - isize
    count, p = X._read_vli(xz, at + 1)
    if count == 0:
        return b"", 0, 0
    assert count == 1
    unpadded, p = X._read_vli(xz, p)
    uncomp, p = X._read_vli(xz, p)
    return xz[12:at], unpadded, uncomp


@pytest.mark.parametrize("check", [0, 1, 4, 10])
@pytest.mark.parametrize("n", [0, 1, 4096, 65537, 300000])
def test_pack_stream_rebuilds_oracle_oneshot_stream(hs, n, check):
    buf = X.gendata("T", n)
    want = X.oracle_buffer_encode(buf, n, 1, check=check)
    block, unpadded, uncomp = _oneshot_block(want)
    assert uncomp == n and len(block) % 4 == 0
    out = (C.c_uint8 * (len(want) + 64))()
    size = hs.bh_pack_stream(block, C.c_uint32(len(block)), C.c_uint64(unpadded), C.c_uint64(uncomp), C.c_uint32(check), out)
    assert size == len(want) and bytes(out[:size]) == want
