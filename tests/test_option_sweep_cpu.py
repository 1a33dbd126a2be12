"""CPU tests (-m "not gpu") of the LZMA2 option sweep of test_gpu_option_sweep.py:
  * the oracle encodes every sweep case to the reference's bytes, and gives the reference decoder's verdict on every
    Stream with a rewritten dictionary size, so it stays a valid stand-in wherever the GPU is compared;
  * the sweep's inputs reach what they are there for: match lists longer than 32 pairs, rep0 matches of 273 bytes,
    overlapping copies over 32 bytes, and matches at exactly the dictionary size."""
import ctypes as C

import pytest

import xzlibs as X
import test_gpu_option_sweep as S

REPS = 4
BACK_LITERAL = 0xFFFFFFFF


def test_oracle_encodes_every_sweep_case_like_the_reference():
    gold = X.ref_golden()["opt_sweep"]
    cases = S.sweep_cases()
    assert len(gold) == len(cases) and 140 <= len(cases) <= 160
    for c in cases:
        assert X.sha64(X.oracle_encode(c.data, len(c.data), 0, c.block_size, c.check, opts=c.opts)) == gold[S.key(c)], S.key(c)


def test_oracle_dict_header_verdicts_match_the_reference():
    """Only the return code: on a data error the oracle delivers no bytes, the reference those before the bad match."""
    gold = X.ref_golden()["dict_header"]
    seen = set()
    for name, o, bs, data in S.dict_header_streams():
        xz = X.oracle_encode(data, len(data), 0, bs, opts=o)
        assert X.sha64(xz) == gold[name]["stream"], name
        for prop in S.DICT_PROPS:
            want = gold[name]["props"][str(prop)]
            r, out = X.oracle_decode(S.set_dict_prop(xz, prop), len(data))
            assert r == want[0], (name, prop, r, want)
            if r == 0:
                assert out == data
            seen.add(r)
    assert seen == {0, 8, 9}   # decodes, LZMA_OPTIONS_ERROR (prop > 40), LZMA_DATA_ERROR (a distance past the dictionary)


def _block_data(case):
    p = 0
    for spec in case.blocks:
        yield spec, case.data[p:p + spec[1]]
        p += spec[1]


def _mf_max_pairs(data, o):
    n = len(data)
    counts = (C.c_uint32 * n)(); longest = (C.c_uint32 * n)(); offs = (C.c_uint64 * n)()
    cap = 64 * n
    while True:
        pairs = (C.c_uint32 * (2 * cap))()
        tot = X.oracle().xzo_mf_dump(data, C.c_uint32(n), C.byref(o), counts, longest, offs, pairs, C.c_uint64(cap), None)
        if tot != 2 ** 64 - 1:
            return max(counts)
        cap *= 4


def _trace(data, o):
    """The oracle's symbols for one Block of `data`: (position, distance, length), distance 0 for a literal, with rep
    matches resolved to their distances."""
    lib = X.oracle()
    cap = len(data) + 16
    tr = (C.c_uint32 * (3 * cap))()
    cnt = C.c_size_t()
    lib.xzo_set_trace(tr, C.c_size_t(cap), C.byref(cnt))
    try:
        X.oracle_encode(data, len(data), 0, len(data), opts=o)
    finally:
        lib.xzo_set_trace(None, C.c_size_t(0), None)
    reps, out = [0, 0, 0, 0], []
    for i in range(cnt.value):
        pos, back, length = tr[3 * i], tr[3 * i + 1], tr[3 * i + 2]
        if back == BACK_LITERAL:
            out.append((pos, 0, 1))
            continue
        if back >= REPS:
            dist = back - REPS
            reps = [dist] + reps[:3]
        else:
            dist = reps[back]
            reps = [dist] + reps[:back] + reps[back + 1:]
        out.append((pos, dist + 1, length))
    return out


def test_ladder_blocks_give_long_match_lists():
    """At nice_len >= 64 the ladder Blocks have positions with more than 32 match pairs: the DP parser's walk past its
    near-candidate fast path and the overflow pool.  A match finder that visits at most 32 nodes cannot list more."""
    n = 0
    for c in S.sweep_cases():
        o = c.opts
        depth = o.depth or (16 + o.nice_len // 2 if o.mf & 0x10 else 4 + o.nice_len // 4)   # the default, lz_encoder.c
        if o.nice_len < 64 or depth <= 32:
            continue
        for spec, data in _block_data(c):
            if spec[0] == "ladder" and len(data) >= 8192:
                assert _mf_max_pairs(data, c.opts) > 32, (c.name, spec)
                n += 1
    assert n >= 40


def test_runs_blocks_give_long_reps_and_overlapping_copies():
    """In every runs Block the oracle codes matches of length 273 and matches with distance < 32 and length > 32."""
    n = 0
    for c in S.sweep_cases():
        for spec, data in _block_data(c):
            if spec[0] != "runs" or len(data) < 8192:
                continue
            syms = _trace(data, c.opts)
            assert any(length == 273 for _, d, length in syms if d), (c.name, spec)
            assert any(d < 32 and length > 32 for _, d, length in syms if d), (c.name, spec)
            n += 1
    assert n >= 100


@pytest.mark.parametrize("mf", [S.HC4, S.BT4])
def test_window_edge_blocks_reach_exactly_the_dictionary(mf):
    """The repeat at gap == dict_size is coded as a match at that distance; the one at dict_size + 1 cannot be."""
    n = 0
    for c in S.sweep_cases():
        if not c.name.startswith("dict-") or c.opts.mf != mf:
            continue
        d = c.opts.dict_size
        for spec, data in _block_data(c):
            gap = spec[2][0]
            far = {dist for _, dist, _ in _trace(data, c.opts) if dist >= d}
            if gap == d:
                assert far == {d}, (c.name, far)
            else:
                assert far == set(), (c.name, gap, far)
            n += 1
    assert n == 18
