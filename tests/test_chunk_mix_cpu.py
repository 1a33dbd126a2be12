"""CPU tests (-m "not gpu") of the chunk-mix cases of tests/chunk_mix.py:
  * the oracle and the host form of the encoder (tests/hostsim) write the reference's Stream for every case and every
    one-shot item (the chunk_mix section of ref_live_golden.json), and so does the live reference where it is built;
  * the cases reach what they are there for, counted from the Blocks' LZMA2 control bytes and the oracle's counters:
    uncompressed -> LZMA switches per mode, per match finder and per lc/lp/pb; uncompressed chunks that swallowed
    read_ahead bytes and are followed by an LZMA chunk, in both modes; a switch in every Block of the coder-warp case;
    an LZMA chunk that ends on the 2 MiB uncompressed limit right before an uncompressed one; LZMA chunks 1-16 bytes
    smaller than their input; one-shot items on both sides of lzma2_bound."""
import ctypes as C
import functools
import os

import pytest

import chunk_mix as M
import xzlibs as X


def gold():
    return X.ref_golden()["chunk_mix"]


@functools.lru_cache(maxsize=1)
def oracle_runs():
    """name -> (Stream, Counters) from the oracle."""
    return {c.name: M.oracle_counters(c) for c in M.cases()}


@pytest.fixture(scope="module")
def hs():
    return C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libhostsim.so"))


def test_oracle_writes_the_reference_stream():
    g = gold()
    assert len(g) == len(M.cases()) + len(M.oneshot_items())
    assert sum(len(c.data) for c in M.cases()) < 48 * M.MiB
    for c in M.cases():
        xz, k = oracle_runs()[c.name]
        want = g[M.key(c)]
        assert X.sha64(xz) == want["stream"], c.name
        assert [k.n_chunks_lzma, k.n_chunks_raw] == list(M.chunk_counts(xz)) == want["chunks"], c.name


def test_hostsim_writes_the_reference_stream(hs):
    for c in M.cases():
        n = len(c.data)
        cap = X.oracle().xzo_stream_bound(n, c.block_size) + 100000
        out = (C.c_uint8 * cap)(); sz = C.c_uint64()
        assert hs.hs_stream_encode(c.data, C.c_uint64(n), C.byref(c.opts), C.c_uint32(c.check), C.c_uint64(c.block_size), out,
                                   C.c_uint64(cap), C.byref(sz)) == 0
        assert X.sha64(out[:sz.value]) == gold()[M.key(c)]["stream"], c.name


@pytest.mark.skipif(not X.have_ref(), reason="oracle/_ref (the unmodified reference) is not built")
def test_live_reference_matches_golden():
    for c in M.cases():
        assert X.sha64(X.ref_encode(c.data, len(c.data), 0, c.block_size, c.check, opts=c.opts)) == gold()[M.key(c)]["stream"], c.name
    for name, p, data in M.oneshot_items():
        assert X.sha64(X.ref_buffer_encode(data, len(data), p)) == gold()[name]["stream"], name


def _switches_by(group):
    out = {}
    for c in M.cases():
        sw = sum(M.switches(b) for b in M.block_chunks(oracle_runs()[c.name][0]))
        k = group(c)
        out[k] = out.get(k, 0) + sw
    return out


def test_switches_in_both_modes_for_every_match_finder_and_lclppb():
    by_mode = _switches_by(lambda c: c.opts.mode)
    assert by_mode[M.FAST] >= 100 and by_mode[M.NORMAL] >= 40, by_mode
    by_mf = _switches_by(lambda c: (c.opts.mode, c.opts.mf))
    for mode in (M.FAST, M.NORMAL):
        for mf in M.MFS:
            assert by_mf.get((mode, mf), 0) >= 2, (mode, hex(mf), by_mf)
    by_lclppb = _switches_by(lambda c: (c.opts.mode, c.opts.lc, c.opts.lp, c.opts.pb))
    for mode in (M.FAST, M.NORMAL):
        for lclppb in M.LCLPPB:
            assert by_lclppb.get((mode, *lclppb), 0) >= 2, (mode, lclppb)
    for p in M.PRESETS:
        assert _switches_by(lambda c: c.name)[f"preset-{M.preset_name(p)}"] >= 2, p


def test_read_ahead_swallowed_then_lzma_in_both_modes():
    """An uncompressed chunk that takes the encoder's read_ahead bytes with it, followed by an LZMA chunk of the same
    Block: the chunk's size includes those bytes, the pending symbols are dropped, and the fast parser restarts after
    them.  Every lazy case has one per Block, for each lc/lp/pb in both modes."""
    per_mode = {M.FAST: 0, M.NORMAL: 0}
    for c in M.cases():
        _, k = oracle_runs()[c.name]
        per_mode[c.opts.mode] += k.n_raw_ahead_then_lzma
        if c.name.startswith("lazy-"):
            assert len(c.blocks) == 2 and k.n_raw_ahead_then_lzma == 2, c.name
    assert per_mode[M.FAST] >= 3 and per_mode[M.NORMAL] >= 3, per_mode
    for mode in (M.FAST, M.NORMAL):
        assert {(c.opts.lc, c.opts.lp, c.opts.pb) for c in M.cases() if c.opts.mode == mode and c.name.startswith("lazy-")} == set(M.LCLPPB)


def test_every_coder_warp_block_switches():
    c = [c for c in M.cases() if c.name == "coderwarp"][0]
    assert c.opts.mode == M.FAST and 16 * M.KiB <= c.block_size <= 64 * M.KiB
    blocks = M.block_chunks(oracle_runs()[c.name][0])
    assert len(blocks) >= 140
    assert all(M.switches(b) >= 1 for b in blocks)


def test_lzma_chunk_ends_on_the_uncompressed_limit_before_an_uncompressed_chunk():
    for c in M.cases():
        if not c.name.startswith("ramp-"):
            continue
        (chunks,) = M.block_chunks(oracle_runs()[c.name][0])
        assert len(c.data) > 2 * M.MiB
        first, second = chunks[0], chunks[1]
        # the chunk stops at the first symbol that reaches 2 MiB - 273, which is where the random bytes start
        assert not M.is_raw(first) and first.usize == M.LZMA2_UNCOMPRESSED_MAX - 273, (c.name, first)
        assert M.is_raw(second) and any(not M.is_raw(ch) for ch in chunks[2:]), (c.name, chunks)


def test_lzma_chunks_just_below_their_input_size():
    """LZMA chunks whose compressed size is 1-16 bytes below their uncompressed size: the edge of the
    `compressed_size >= uncompressed_size` test that picks the chunk kind."""
    near = 0
    for c in M.cases():
        for b in M.block_chunks(oracle_runs()[c.name][0]):
            near += sum(1 for ch in b if not M.is_raw(ch) and 1 <= ch.usize - ch.csize <= 16)
    assert near >= 5


def test_oneshot_items_on_both_sides_of_the_bound(hs):
    """lzma_easy_buffer_encode keeps its LZMA2 data only if it fits lzma2_bound(n), else it writes an uncompressed
    Block (block_buffer_encoder.c): items from 3 bytes under to 2 bytes over the bound, at -0 and -6."""
    class Res(C.Structure):
        _fields_ = [("total_size", C.c_uint32), ("header_size", C.c_uint32), ("unpadded_size", C.c_uint64), ("fallback", C.c_uint32),
                    ("ret", C.c_uint32), ("n_symbols", C.c_uint32), ("n_chunks_lzma", C.c_uint32), ("n_chunks_raw", C.c_uint32), ("pad_", C.c_uint32)]
    seen = {0: set(), 6: set()}
    for name, p, data in M.oneshot_items():
        n = len(data)
        d = M.oneshot_lzma2_size(data, p) - M.lzma2_bound(n)
        seen[p].add(d)
        xz = X.oracle_buffer_encode(data, n, p)
        assert X.sha64(xz) == gold()[name]["stream"], name
        # the uncompressed fallback announces LZMA_DICT_SIZE_MIN (property 0); presets 0 and 6 use 256 KiB and 8 MiB
        assert (M.dict_prop(xz, 12) == 0) == (d > 0), (name, d)
        out = (C.c_uint8 * (len(xz) + 200000))(); res = Res()   # room for a whole LZMA2 chunk
        assert hs.hs_block_encode(data, C.c_uint32(n), C.byref(X.preset_options(p)), C.c_uint32(4), C.c_uint64(0), out,
                                  C.c_uint32(len(out)), C.byref(res)) == 0
        assert bytes(out[:res.total_size]) == xz[12:12 + res.total_size], name
    for p in seen:
        assert set(range(-3, 3)) <= seen[p], (p, seen[p])
