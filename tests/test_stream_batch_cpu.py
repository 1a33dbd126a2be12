"""CPU tests of the whole-Stream batch encoder's host pieces (xzb_stream_encode_batch), compiled by
tests/hostsim/batch_host.cpp (the planner) and tests/hostsim/stream_batch_host.cpp (placement and packing):
  * the wave planner (xz_b200/csrc/xzb_params.h) on per-Block size lists of whole-Stream items: every Block's
    predecessors in its item are in its wave or an earlier one, in Block order, which Block placement relies on;
  * Stream placement and the multi-Block Stream packing that xzb_k_pack_streams runs
    (xzb_pack_block, xz_b200/csrc/xzb_frame.cuh): the Blocks of an oracle lzma_stream_encoder_mt Stream, placed and framed again piece
    by piece, in one wave and in several, are that Stream byte for byte; a slot too small fails alone."""
import ctypes as C
import os
import random
import types

import pytest

import chunk_mix as M
import xzlibs as X
from test_oracle import STREAM_CASES

KiB, MiB = 1 << 10, 1 << 20
BUF_ERROR = 10


@pytest.fixture(scope="module")
def hs():
    plan = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libbatchhost.so"))
    plan.bh_plan_waves.restype = C.c_uint32
    pack = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libstreambatchhost.so"))
    pack.bh_pack_waves.restype = C.c_uint32
    return types.SimpleNamespace(bh_plan_waves=plan.bh_plan_waves, bh_pack_waves=pack.bh_pack_waves)


def _blocks_of(in_sizes, bs):
    """(item, j, size) of every Block, in (item, j) order, as the batch driver lists them."""
    out = []
    for i, n in enumerate(in_sizes):
        for j in range((n + bs - 1) // bs):
            out.append((i, j, min(bs, n - j * bs)))
    return out


def _plan(hs, sizes, per_byte, per_block, budget, hash_bits, max_blocks):
    n = len(sizes)
    A = C.c_uint32 * max(n, 1)
    order, wave, off = A(), A(), A()
    nw = hs.bh_plan_waves((C.c_uint64 * max(n, 1))(*sizes), C.c_uint32(n), C.c_uint64(per_byte), C.c_uint64(per_block),
                          C.c_uint64(budget), C.c_uint32(hash_bits), C.c_uint32(max_blocks), order, wave, off)
    return nw, [(order[k], wave[k]) for k in range(n)]


@pytest.mark.parametrize("max_blocks", [1, 3, 7, 0])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_planner_keeps_each_items_blocks_in_order(hs, seed, max_blocks):
    """Items of many full Blocks plus a short tail, of exactly k Blocks, shorter than one Block, and empty; budgets
    from a few Blocks per wave to all of them."""
    rng = random.Random(seed)
    bs = rng.choice((64 * KiB, MiB, 3 * MiB))
    in_sizes = []
    for _ in range(60):
        shape = rng.randrange(5)
        k = rng.randrange(1, 12)
        in_sizes.append((0, k * bs, k * bs + rng.randrange(1, bs), rng.randrange(1, bs), bs - 1)[shape])
    blocks = _blocks_of(in_sizes, bs)
    sizes = [s for _, _, s in blocks]
    per_byte, per_block = 130, 75000
    for budget in (per_byte * 2 * bs + 3 * per_block, per_byte * 9 * bs, 1 << 40):
        nw, placed = _plan(hs, sizes, per_byte, per_block, budget, 22, max_blocks)
        assert sorted(k for k, _ in placed) == list(range(len(blocks)))
        wave_of = {k: w for k, w in placed}
        pos_of = {k: p for p, (k, _) in enumerate(placed)}
        for k, (i, j, _) in enumerate(blocks):
            if j > 0:
                prev = k - 1
                assert wave_of[prev] <= wave_of[k], (i, j)
                assert pos_of[prev] < pos_of[k], (i, j)   # within a wave too: placement walks it in this order
        if max_blocks:
            assert all(sum(1 for _, w in placed if w == x) <= max_blocks for x in range(nw))
        if budget < 1 << 40 or max_blocks:
            assert nw > 1


def _cut(xz, bs, n):
    """(Blocks, Index records) of an lzma_stream_encoder_mt Stream of n bytes in Blocks of bs."""
    unpadded = M._index_records(xz)
    assert len(unpadded) == (n + bs - 1) // bs
    blocks, at = [], 12
    for j, u in enumerate(unpadded):
        total = (u + 3) & ~3
        blocks.append((xz[at: at + total], u, min(bs, n - j * bs)))
        at += total
    return blocks


def _pack(hs, streams, waves_of, check, nthreads, caps=None):
    """Rebuild the Streams [(Blocks, ...)] through bh_pack_waves; waves_of(k) is the wave of the k-th Block overall."""
    n = len(streams)
    flat = [b for s in streams for b in s]
    data = b"".join(b for b, _, _ in flat)
    boff, at = [], 0
    for b, _, _ in flat:
        boff.append(at)
        at += len(b)
    caps = caps or [12 + sum(len(b) for b, _, _ in s) + 8 + 18 * len(s) + 12 + 64 for s in streams]
    offs = [0]
    for c in caps[:-1]:
        offs.append(offs[-1] + c + 3)  # unaligned slots with gaps between them
    total = offs[-1] + caps[-1] + 3 if n else 1
    out = (C.c_uint8 * total)(*([0xA5] * total))
    A64, A32 = C.c_uint64 * max(n, 1), C.c_uint32 * max(n, 1)
    B64, B32 = C.c_uint64 * max(len(flat), 1), C.c_uint32 * max(len(flat), 1)
    size, ret = A64(), A32()
    src = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    nw = hs.bh_pack_waves(C.c_uint32(n), A64(*[len(s) for s in streams]), src, B64(*boff), B32(*[len(b) for b, _, _ in flat]),
                          B64(*[u for _, u, _ in flat]), B64(*[v for _, _, v in flat]), B32(*[waves_of(k) for k in range(len(flat))]),
                          C.c_uint32(check), C.c_uint32(nthreads), out, A64(*offs), A64(*caps), size, ret)
    assert nw != 0xFFFFFFFF
    raw = bytes(out)
    return [(ret[i], raw[offs[i]: offs[i] + size[i]]) for i in range(n)], raw, offs, caps


@pytest.mark.parametrize("check", [0, 1, 4, 10])
def test_pack_waves_rebuild_oracle_mt_streams(hs, check):
    """The oracle's lzma_stream_encoder_mt Streams for the STREAM_CASES sizes, plus the Stream with no Block, cut into
    Blocks and Index records and fed back: all in one wave, one Block per wave, and in waves of three; 1 and 7 workers."""
    streams, want = [], []
    for preset, n, bs in STREAM_CASES:
        xz = X.oracle_encode(X.gendata("T", n), n, preset, bs, check=check)
        want.append(xz)
        streams.append(_cut(xz, bs, n))
    empty = X.oracle_encode(X.gendata("T", 0), 0, 6, MiB, check=check)
    assert len(empty) == 32
    want.append(empty)
    streams.append([])
    for waves_of in (lambda k: 0, lambda k: k, lambda k: k // 3):
        for nthreads in (1, 7):
            got, raw, offs, caps = _pack(hs, streams, waves_of, check, nthreads)
            assert [r for r, _ in got] == [0] * len(want)
            assert [xz for _, xz in got] == want
            # nothing outside the Streams was written
            ends = [o + len(w) for o, w in zip(offs, want)]
            assert all(b == 0xA5 for b in raw[:offs[0]])
            for i in range(len(want) - 1):
                assert set(raw[ends[i]: offs[i + 1]]) <= {0xA5}


def test_pack_waves_slot_one_byte_short_fails_alone(hs):
    preset, n, bs = STREAM_CASES[0]
    xz = X.oracle_encode(X.gendata("E", n), n, preset, bs)
    s = _cut(xz, bs, n)
    empty = X.oracle_encode(X.gendata("E", 0), 0, preset, bs)
    for short in (0, 1):   # the short item is the multi-Block one, then the one with no Block
        caps = [len(xz), len(empty), len(xz)]
        caps[short] -= 1
        got, _, _, _ = _pack(hs, [s, [], s], lambda k: k // 2, 4, 3, caps)
        want = [(0, xz), (0, empty), (0, xz)]
        want[short] = (BUF_ERROR, b"")
        assert got == want
