"""Seeded inputs that make the LZMA2 chunker switch between LZMA and uncompressed chunks inside one Block, and the case
list of test_chunk_mix_cpu.py / test_gpu_chunk_mix.py.  Only hashes are stored (the chunk_mix section of
tests/golden/ref_live_golden.json); the inputs are made here.

When an LZMA attempt compresses to no less than its input, lzma2_encode writes the chunk uncompressed, resets the LZMA
state (probabilities, reps, price counters, pending optimum symbols), swallows the encoder's read_ahead bytes into the
uncompressed chunk without advancing the position that selects pos_state and the literal coder (SURVEY D12), and
marks the next LZMA chunk with a state reset (control byte 0xA0).  None of that changes the decoded bytes of a wrong
encoder, only the encoded ones, so these cases are compared byte for byte with the reference.

Generators:
  marginal  random bytes plus sparse 2-8-byte copies at distances 1-64, the copy rate redrawn every 32 KiB around the
            rate where LZMA just stops paying: chunk after chunk flips between the two kinds;
  patchy    random stretches of 1-150 KB alternating with text stretches;
  lazy      random bytes, a zone of "lazy" spots (a 3-byte match at a short distance, then a 6-byte match one position
            later, so the parser codes a literal and keeps the next position's match: read_ahead = 1) around where the
            first chunk fills its 64 KiB of output, then text.  LAZY_SEEDS are seeds where that chunk is uncompressed,
            ends with read_ahead > 0 and the next chunk is LZMA (found by search_lazy(), run offline);
  tailed    one 64 KiB Block: random bytes, then zeros: an uncompressed chunk that fills 64 KiB, then an LZMA chunk;
  ramp      a short-period pattern up to the 2 MiB uncompressed limit of an LZMA chunk (less the longest match), then
            random bytes, then text.
"""
import functools
import random
import struct
from collections import namedtuple

import xzlibs as X

KiB, MiB = 1 << 10, 1 << 20
HC3, HC4, BT2, BT3, BT4 = 0x03, 0x04, 0x12, 0x13, 0x14
MFS = (HC3, HC4, BT2, BT3, BT4)
FAST, NORMAL = 1, 2
CHECK_SHA256 = 10
CHECKS = (X.CHECK_NONE, X.CHECK_CRC32, X.CHECK_CRC64, CHECK_SHA256)
PRESETS = (0, 1, 2, 3, 4, 6, 9 | X.XZ_PRESET_EXTREME)
LCLPPB = ((3, 0, 2), (0, 4, 4), (4, 0, 4), (1, 3, 1), (3, 0, 0))
LAZY_N = 72 * KiB
LZMA2_CHUNK_MAX = 1 << 16
LZMA2_UNCOMPRESSED_MAX = 1 << 21

# (mode, lc, lp, pb) -> seeds of lazy() Blocks whose first, uncompressed chunk ends with read_ahead > 0 and is followed
# by an LZMA chunk; from search_lazy(opts_for(mode, lc, lp, pb), 2)
LAZY_SEEDS = {
    (FAST, 3, 0, 2): (25, 48), (FAST, 0, 4, 4): (32, 43), (FAST, 4, 0, 4): (33, 47), (FAST, 1, 3, 1): (19, 31),
    (FAST, 3, 0, 0): (14, 27),
    (NORMAL, 3, 0, 2): (40, 66), (NORMAL, 0, 4, 4): (9, 12), (NORMAL, 4, 0, 4): (34, 44), (NORMAL, 1, 3, 1): (11, 26),
    (NORMAL, 3, 0, 0): (25, 35),
}

# (preset, seed, n, copy rate) of marginal() one-shot items whose LZMA2 data ends within a few bytes of
# lzma2_bound(n), on both sides; from search_oneshot()
ONESHOT = ((0, 0, 2000, 0.004), (0, 363, 3911, 0.01), (0, 906, 5282, 0.006), (0, 1032, 10904, 0.008),
           (0, 1151, 9547, 0.006), (0, 1552, 49344, 0.008),
           (6, 0, 2000, 0.004), (6, 2, 3994, 0.008), (6, 121, 2637, 0.006), (6, 142, 23574, 0.008),
           (6, 545, 5365, 0.004), (6, 726, 5822, 0.006))

# name: unique label; blocks: the generator of each Block, in order (the input is their concatenation)
Case = namedtuple("Case", "name opts check block_size blocks data")


# ---- input generators ----

def marginal(n, seed, rate=0.0052, stretch=32 * KiB, spread=0.5):
    rnd = random.Random(seed)
    out = bytearray(rnd.randbytes(64))
    while len(out) < n:
        end = len(out) + stretch
        q = rate * (1 + spread * (2 * rnd.random() - 1))
        while len(out) < end:
            out += rnd.randbytes(int(rnd.expovariate(q)))
            length, dist = rnd.randint(2, 8), rnd.randint(1, 64)
            for _ in range(length):
                out.append(out[-dist])
    return bytes(out[:n])


def patchy(n, seed):
    rnd = random.Random(seed)
    out = bytearray()
    while len(out) < n:
        k = rnd.randint(1000, 150000)
        out += rnd.randbytes(k) if rnd.random() < 0.5 else bytes(X.gendata("T", k, len(out))[:k])
    return bytes(out[:n])


def lazy(n, seed, zone=(60000, 68000), every=24, tail=4096):
    rnd = random.Random(seed)
    out = bytearray(rnd.randbytes(n - tail)) + bytes(X.gendata("T", tail, seed)[:tail])
    x = zone[0]
    while x + 8 < zone[1]:
        far, near = rnd.randint(200, 4000), rnd.randint(1, 64)
        out[x + 1:x + 7] = out[x + 1 - far:x + 7 - far]   # 6-byte match at x + 1
        out[x - near:x - near + 3] = out[x:x + 3]          # 3-byte match at x
        x += rnd.randint(every // 2, every * 3 // 2)
    return bytes(out)


def tailed(n, seed, zeros=256):
    return random.Random(seed).randbytes(n - zeros) + bytes(zeros)


def ramp(n, seed, head=LZMA2_UNCOMPRESSED_MAX - 273, noise=256 * KiB):
    assert n > head + noise
    rnd = random.Random(seed)
    unit = rnd.randbytes(61)
    out = (unit * (head // len(unit) + 1))[:head] + rnd.randbytes(noise)
    return (out + bytes(X.gendata("T", n - len(out), seed)[:n - len(out)]))[:n]


GENS = {"marginal": marginal, "patchy": patchy, "lazy": lazy, "tailed": tailed, "ramp": ramp}


def make_block(spec):
    kind, n, seed = spec
    return GENS[kind](n, seed)


# ---- the cases ----

def opts_for(mode, lc=3, lp=0, pb=2, mf=None, nice=None, dict_size=8 * MiB):
    mf = mf if mf is not None else (HC4 if mode == FAST else BT4)
    nice = nice if nice is not None else (273 if mode == FAST else 64)
    return X.LzmaOptions(dict_size, lc, lp, pb, mode, nice, mf, 0)


def preset_name(p):
    return "9e" if p & X.XZ_PRESET_EXTREME else str(p)


@functools.lru_cache(maxsize=1)
def cases():
    raw = []   # (name, opts, block_size, block specs)
    for i, p in enumerate(PRESETS):
        raw.append((f"preset-{preset_name(p)}", X.preset_options(p), 512 * KiB, [("marginal", 512 * KiB, 100 + 3 * i + b) for b in range(3)]))
    for mode in (FAST, NORMAL):
        for mf in MFS:
            nice = 273 if mode == FAST else 64
            raw.append((f"mf-{mode}-{mf:x}", opts_for(mode, mf=mf, nice=nice), 512 * KiB,
                        [("marginal", 512 * KiB, 200 + 10 * mode + mf + b) for b in range(2)]))
    for mode in (FAST, NORMAL):
        for lc, lp, pb in LCLPPB:
            seeds = LAZY_SEEDS.get((mode, lc, lp, pb), ())
            raw.append((f"lazy-{mode}-{lc}{lp}{pb}", opts_for(mode, lc, lp, pb), LAZY_N, [("lazy", LAZY_N, s) for s in seeds]))
    for p in (0, 6):
        raw.append((f"patchy-{p}", X.preset_options(p), 2 * MiB, [("patchy", 2 * MiB, 300 + p), ("patchy", MiB + 4321, 301 + p)]))
    for mode in (FAST, NORMAL):
        raw.append((f"ramp-{mode}", opts_for(mode), 4 * MiB, [("ramp", 3 * MiB, 400 + mode)]))
    # the coder-warp form of the fast kernel: a wave with more Blocks than the H100's 132 SMs
    raw.append(("coderwarp", opts_for(FAST), 64 * KiB, [("tailed", 64 * KiB, 500 + b) for b in range(144)]))
    out = []
    for i, (name, o, bs, specs) in enumerate(raw):
        data = b"".join(make_block(s) for s in specs)
        out.append(Case(name, o, CHECKS[i % 4], bs, tuple(specs), data))
    return tuple(out)


def key(case):
    o = case.opts
    return f"{case.name}|{o.mode}.{o.mf:x}.{o.nice_len}.{o.depth}.{o.dict_size}.{o.lc}{o.lp}{o.pb}|{case.check}|{case.block_size}|{len(case.data)}"


@functools.lru_cache(maxsize=1)
def oneshot_items():
    """(name, preset, input) of the one-shot items."""
    return tuple((f"oneshot-{preset_name(p)}-{seed}-{n}", p, marginal(n, seed, rate)) for p, seed, n, rate in ONESHOT)


def lzma2_bound(n):
    """lzma2_bound (block_buffer_encoder.c): the most LZMA2 data lzma_block_buffer_encode keeps before it falls back to
    an uncompressed Block."""
    return n + (n + LZMA2_CHUNK_MAX - 1) // LZMA2_CHUNK_MAX * 3 + 1


# ---- reading the chunks back ----

Chunk = namedtuple("Chunk", "control usize csize")   # csize = usize for an uncompressed chunk


def _index_records(xz):
    back = (struct.unpack_from("<I", xz, len(xz) - 8)[0] + 1) * 4
    count, p = X._read_vli(xz, len(xz) - 12 - back + 1)
    recs = []
    for _ in range(count):
        unpadded, p = X._read_vli(xz, p)
        _, p = X._read_vli(xz, p)
        recs.append(unpadded)
    return recs


def lzma2_chunks(data, pos=0):
    """The chunks of one LZMA2 stream starting at data[pos], up to its end marker, and the end marker's position + 1."""
    chunks = []
    while True:
        c = data[pos]
        if c == 0:
            return chunks, pos + 1
        if c in (1, 2):
            u = (data[pos + 1] << 8 | data[pos + 2]) + 1
            chunks.append(Chunk(c, u, u))
            pos += 3 + u
            continue
        assert c >= 0x80, c
        u = ((c & 0x1F) << 16 | data[pos + 1] << 8 | data[pos + 2]) + 1
        s = (data[pos + 3] << 8 | data[pos + 4]) + 1
        chunks.append(Chunk(c, u, s))
        pos += 5 + (c >= 0xC0) + s


def dict_prop(xz, pos):
    """The LZMA2 dictionary property of the Block Header at xz[pos]."""
    flags, q = xz[pos + 1], pos + 2
    for bit in (0x40, 0x80):
        if flags & bit:
            _, q = X._read_vli(xz, q)
    assert xz[q] == 0x21 and xz[q + 1] == 1
    return xz[q + 2]


def block_chunks(xz):
    """[chunks of each Block] of a one-Stream .xz file."""
    out, pos = [], 12
    for unpadded in _index_records(xz):
        hs = (xz[pos] + 1) * 4
        chunks, end = lzma2_chunks(xz, pos + hs)
        out.append(chunks)
        pos += (unpadded + 3) & ~3
    return out


def is_raw(ch):
    return ch.control < 0x80


def switches(chunks):
    """Uncompressed -> LZMA switches inside one Block."""
    return sum(1 for a, b in zip(chunks, chunks[1:]) if is_raw(a) and not is_raw(b))


def chunk_counts(xz):
    """(LZMA chunks, uncompressed chunks) over all Blocks."""
    allc = [c for b in block_chunks(xz) for c in b]
    raw = sum(1 for c in allc if is_raw(c))
    return len(allc) - raw, raw


def oracle_counters(case):
    c = X.Counters()
    xz = X.oracle_encode(case.data, len(case.data), 0, case.block_size, case.check, opts=case.opts, counters=c)
    return xz, c


# ---- the searches that picked LAZY_SEEDS and ONESHOT (python tests/chunk_mix.py) ----

def search_lazy(o, count, start=0):
    seeds, seed = [], start
    while len(seeds) < count:
        c = X.Counters()
        X.oracle_encode(lazy(LAZY_N, seed), LAZY_N, 0, LAZY_N, opts=o, counters=c)
        if c.n_raw_ahead_then_lzma:
            seeds.append(seed)
        seed += 1
    return seeds


def oneshot_lzma2_size(data, preset):
    """Size of the LZMA2 data lzma_block_buffer_encode makes before its fit test: the mt framing's Block with the
    same LZMA2 stream."""
    xz = X.oracle_encode(data, len(data), preset, max(len(data), 1))
    _, end = lzma2_chunks(xz, 12 + (xz[12] + 1) * 4)
    return end - 12 - (xz[12] + 1) * 4


def search_oneshot(presets=(0, 6), deltas=range(-3, 3)):
    """For each preset and each LZMA2 size - lzma2_bound(n) in deltas, one (preset, seed, n, rate)."""
    found = []
    for p in presets:
        want = set(deltas)
        seed = 0
        while want:
            n = 2000 + seed * 997 % 60000
            rate = 0.004 + 0.002 * (seed % 5)
            d = oneshot_lzma2_size(marginal(n, seed, rate), p) - lzma2_bound(n)
            if d in want:
                want.discard(d)
                found.append((p, seed, n, rate))
            seed += 1
    return found


if __name__ == "__main__":
    print("LAZY_SEEDS = {")
    for mode in (FAST, NORMAL):
        for lc, lp, pb in LCLPPB:
            print(f"    ({mode}, {lc}, {lp}, {pb}): {tuple(search_lazy(opts_for(mode, lc, lp, pb), 2))},", flush=True)
    print("}")
    print("ONESHOT =", tuple(search_oneshot()))
