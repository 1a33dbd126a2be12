"""CPU tests of the LZMA2 decoders on the generated Streams of tests/lzma2_gen.py: valid input that an LZMA2 encoder
byte-identical to liblzma's never writes (mid-Block dictionary and state resets, new lc/lp/pb, 0x80 after an
uncompressed chunk, 1-byte and maximal chunks, far length-2 matches, distances at the window's edge, empty Blocks)
and a few near misses one step past an edge.  Each case carries its plaintext by construction; the reference's answers
on its Streams are recorded in ref_live_golden.json (section lzma2_gen) and checked live where oracle/_ref is built.

The oracle (xzo_lzma2_decode) and the host form of the product's decoder (xzb_dec.cuh, through tests/hostsim) must give
the plaintext on every valid payload and the reference's verdict on every near miss."""
import ctypes as C
import os

import pytest

import lzma2_gen as G
import xzlibs as X


@pytest.fixture(scope="module")
def hs():
    return C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libhostsim.so"))


def _ids(cases):
    return [c.name for c in cases]


CASES = G.cases()


@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_generator_matches_recorded_reference(case):
    """The generator's plaintext and verdict are the reference decoder's recorded answer, single-threaded, threaded and
    on the unsized Block (a changed generator must be re-recorded on purpose)."""
    g = X.ref_golden()["lzma2_gen"][case.name]
    assert g["stream"] == X.sha64(case.xz)
    for r, size, digest in g["decode"]:
        assert r == case.verdict
        if case.verdict == 0:
            assert [size, digest] == [len(case.expected), X.sha64(case.expected)]


def _verdict(r):
    """need-input / need-output (100 / 101 from the host form, XZO_BUF_ERROR from the oracle) are LZMA_BUF_ERROR."""
    return 10 if r in (100, 101) else r


@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_oracle_and_host_decoder_on_raw_payload(hs, case):
    n = max(case.declared, 1)
    out = (C.c_uint8 * n)(); osz = C.c_size_t(); iu = C.c_size_t()
    ro = X.oracle().xzo_lzma2_decode(case.payload, C.c_size_t(len(case.payload)), C.c_uint32(case.dict_size), out, C.c_size_t(case.declared),
                                     C.byref(osz), C.byref(iu))
    hout = (C.c_uint8 * n)(); hiu = C.c_uint32(); hou = C.c_uint32()
    rh = hs.hs_lzma2_decode(case.payload, C.c_uint32(len(case.payload)), C.c_uint32(case.dict_size), hout, C.c_uint32(case.declared),
                            C.byref(hiu), C.byref(hou))
    assert _verdict(ro) == case.verdict and _verdict(rh) == case.verdict
    if case.verdict == 0:
        assert iu.value == hiu.value == len(case.payload)
        assert bytes(out[:osz.value]) == case.expected
        assert bytes(hout[:hou.value]) == case.expected


@pytest.mark.skipif(not X.have_ref(), reason="oracle/_ref is not built")
@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_live_reference(case):
    for xz in (case.xz, X.drop_block_sizes(case.xz)):
        r, back = X.ref_decode(xz, case.declared)
        assert r == case.verdict
        if case.verdict == 0:
            assert back == case.expected


def test_coverage():
    """What the cases emit: every (state, symbol kind); every distance slot up to the farthest match the biggest Block
    allows; every match and rep length 2..273; every control-byte transition a valid payload can have; LZMA chunks and
    mid-Block dictionary resets at every position modulo 16; all 75 lc/lp/pb; the warp decoder's copy geometries and
    the window edges."""
    cov = G.coverage()
    assert cov.state_kind == {(s, k) for s in range(12) for k in G.KINDS}
    big = next(c for c in CASES if c.name == "big")
    top = G.dist_slot(len(big.expected) - 273 - 1)     # the Block ends on a 273-byte match from its first byte
    assert top >= 51
    assert {s for _, s in cov.slots} == set(range(top + 1))
    assert {s for lps, s in cov.slots if lps == 0} == set(range(top + 1)), "length-2 matches at every distance"
    assert cov.match_lens == cov.rep_lens == set(range(2, 274))
    assert cov.transitions == G.valid_transitions()
    assert cov.lzma_start_mod16 == cov.reset_mod16 == set(range(16))
    assert cov.props == set(G.PROPS)
    for ev in G.GEOMETRY_EVENTS + G.WINDOW_EVENTS:
        assert cov.events[ev] > 0, ev
    sizes = {}
    for c in CASES:
        p, i = c.payload, 0
        while p[i]:
            lz = p[i] >= 0x80
            u = ((p[i] & 0x1F) << 16 | p[i + 1] << 8 | p[i + 2]) + 1 if lz else (p[i + 1] << 8 | p[i + 2]) + 1
            cs = (p[i + 3] << 8 | p[i + 4]) + 1 if lz else u
            sizes.setdefault(lz, set()).add(u)
            i += (6 if p[i] >= 0xC0 else 5 if lz else 3) + cs
    assert {1, 2 * G.MiB} <= sizes[True] and {1, 65536} <= sizes[False]
    assert sum(c.verdict == 0 and not c.expected for c in CASES) == 1       # the end-marker-only Block
    assert len(big.expected) > 80 * 10 ** 6
    hr = next(c for c in CASES if c.name == "high_ratio")
    assert len(hr.expected) >= 16 * G.MiB and len(hr.payload) < 100 * 1024


def test_crc64_equals_oracle():
    data = bytes(X.gendata("E", 100003)[:100003])
    for n in (0, 1, 7, 8, 9, 100003):
        assert G.crc64(data[:n]) == X.oracle().xzo_crc64(data[:n], n, 0)


def test_generator_is_deterministic():
    """Identical cases from a second run of the families (splitmix64 and SHAKE-128 only)."""
    again = G._symbol_mix(G.Coverage()) + G._window_edge(G.Coverage())
    first = {c.name: c for c in CASES}
    for c in again:
        assert c == first[c.name]
