"""The normal-mode parser's "literal + rep0" candidate (lzma_encoder_optimum_normal.c:562-597) against the oracle.

The worker that owns a DP node pushes this candidate last, once the chain warp has decided slot c+1, while the gather
warp holds only the one slot it lands on.  The inputs are seeded and built so that the candidate is common and often
wins:
  subst  copies from one distance with one-byte substitutions, each followed by a tail of 2 .. 7, 9 .. 40 bytes that
         still matches at that distance (the candidate lands on c+3 .. c+41);
  rare   the same substitution behind a copy, where another, older distance matches the substituted byte and the next
         40 bytes: the node has a match of 41 bytes, so its worker takes the path for uncommon shapes.
In the `subst` inputs at nice_len 8 and 5 the pushed "literal + rep0" is, at least once, the only thing that carries the
DP segment past c+1 (so the late raise of len_end decides where the segment ends; counted by the XZB_DP_PROF build).
Presets -6 (nice_len 64, 12 workers) and -9e (nice_len 273: 3 workers, 1024-entry rings), and -6 with nice_len 8 (the
shortest with the near wave) and 5 (no near wave).
"""
import ctypes as C
import random

import pytest

import xzlibs as X

N = 3 << 17
BLOCK = 1 << 18
BACK_LITERAL = 0xFFFFFFFF
TAILS = (2, 3, 4, 5, 6, 7, 9, 12, 20, 40)


def subst(n, seed):
    rnd = random.Random(seed)
    out = bytearray(rnd.randbytes(2048))
    while len(out) < n:
        d = rnd.randint(8, 1500)
        for _ in range(rnd.randint(6, 40)):
            out.append(out[-d])
        for _ in range(rnd.randint(1, 4)):
            out.append(out[-d] ^ rnd.randint(1, 255))
            for _ in range(rnd.choice(TAILS)):
                out.append(out[-d])
        out += rnd.randbytes(rnd.randint(0, 12))
    return bytes(out[:n])


def rare(n, seed):
    rnd = random.Random(seed)
    out = bytearray(rnd.randbytes(4096))
    while len(out) < n:
        r0 = len(out) - rnd.randint(300, 1500)
        x = out[r0 - 1] ^ rnd.randint(1, 255)
        out.append(x)                       # the template: x and the 40 bytes at r0
        out += out[r0:r0 + 40]
        out += rnd.randbytes(rnd.randint(20, 200))
        m = rnd.randint(4, 20)
        d = len(out) + m + 1 - r0           # the copy ends right before r0 - 1 recurs, where x stands instead
        for _ in range(m):
            out.append(out[-d])
        out.append(x)
        for _ in range(rnd.choice(TAILS)):
            out.append(out[-d])
        out += rnd.randbytes(rnd.randint(0, 30))
    return bytes(out[:n])


GENS = {"subst": subst, "rare": rare}
# (label, preset, nice_len or None for the preset's)
SETTINGS = (("-6", 6, None), ("-9e", 0x80000009, None), ("-6 nice 8", 6, 8), ("-6 nice 5", 6, 5))
CASES = [(g, s, seed) for g in GENS for s in SETTINGS for seed in (1, 2)]


def _opts(preset, nice):
    o = X.preset_options(preset)
    if nice is not None:
        o.nice_len = nice
    return o


def _case_id(case):
    g, (label, _, _), seed = case
    return f"{g}-{label.replace(' ', '')}-{seed}"


def _lit_rep0_pairs(data, o):
    """Literals that the oracle's parse follows directly with a rep0 match of 2 bytes or more."""
    lib = X.oracle()
    cap = len(data) + 16
    tr = (C.c_uint32 * (3 * cap))()
    cnt = C.c_size_t()
    lib.xzo_set_trace(tr, C.c_size_t(cap), C.byref(cnt))
    try:
        X.oracle_encode(data, len(data), 0, BLOCK, opts=o)
    finally:
        lib.xzo_set_trace(None, C.c_size_t(0), None)
    pairs, prev = 0, None
    for i in range(cnt.value):
        pos, back, length = tr[3 * i], tr[3 * i + 1], tr[3 * i + 2]
        if prev is not None and prev[1] == BACK_LITERAL and prev[0] + 1 == pos and back == 0 and length >= 2:
            pairs += 1
        prev = (pos, back)
    return pairs


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_inputs_have_literal_rep0_pairs(case):
    """Each input really makes the parser choose "literal + rep0" (so the GPU comparison cannot pass vacuously)."""
    g, (_, preset, nice), seed = case
    data = GENS[g](N, seed)
    assert _lit_rep0_pairs(data, _opts(preset, nice)) >= 100


@pytest.fixture(scope="module")
def ctx():
    import xz_b200
    c = xz_b200.Context(0)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_lit_rep0_inputs_match_oracle(ctx, case):
    import xz_b200
    g, (_, preset, nice), seed = case
    data = GENS[g](N, seed)
    o = _opts(preset, nice)
    po = xz_b200.LzmaOptions(*(getattr(o, f) for f, _ in X.LzmaOptions._fields_))
    mine = ctx.stream_encode(data, opts=po, block_size=BLOCK, n=N)
    assert mine == X.oracle_encode(data, N, 0, BLOCK, opts=o)
    r, back = ctx.stream_decode(mine, N)
    assert r == 0 and back == data
