"""An independent LZMA / LZMA2 encoder of chosen symbols, for testing the decoders on valid input that an LZMA2 encoder
byte-identical to liblzma's never writes (test helper, not a test module).

Written from the format (the LZMA range coder, its adaptive bit model, bit trees, reverse bit trees and direct bits;
the LZMA2 chunk headers; the .xz Stream, Block Header, Index and Footer), not from any encoder's sources.  Nothing here
searches for matches: a seeded splitmix64 generator picks each symbol -- literal, match, short rep, rep0..rep3 with
a distance and a length -- and the generator applies it to its own output buffer.  Every case so carries its expected
plaintext by construction, and the same seeds give the same bytes on every machine and Python version.

cases() returns the case list; coverage() what the cases emitted (state x symbol kind, distance slots, lengths,
control-byte transitions, copy geometries of the GPU decoder's warp form, window edges) for the coverage assertions of
tests/test_lzma2_gen_cpu.py.  tests/golden/make_ref_golden.py records the reference decoder's answers on the Streams.
"""
import collections
import hashlib
import struct
import zlib

M64 = (1 << 64) - 1
DATA_ERROR = 9        # LZMA_DATA_ERROR == XZB_DATA_ERROR == XZO_DATA_ERROR
MiB = 1 << 20
KINDS = ("lit", "match", "short", "rep0", "rep1", "rep2", "rep3")
LZMA_CTRL = (0x80, 0xA0, 0xC0, 0xE0)
PROPS = [(lc, lp, pb) for pb in range(5) for lc in range(5) for lp in range(5) if lc + lp <= 4]   # 75 combinations


class Rng:
    """splitmix64."""

    def __init__(self, seed):
        self.s = seed & M64

    def next(self):
        self.s = (self.s + 0x9E3779B97F4A7C15) & M64
        z = self.s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        return z ^ (z >> 31)

    def below(self, n):
        return self.next() % n

    def between(self, a, b):
        """Uniform in [a, b]."""
        return a + self.next() % (b - a + 1)

    def pick(self, weighted):
        """One key of [(key, weight), ...]."""
        r = self.below(sum(w for _, w in weighted))
        for k, w in weighted:
            if r < w:
                return k
            r -= w
        raise AssertionError

    def log_between(self, a, b):
        """Roughly log-uniform in [a, b]."""
        hi = self.between(a.bit_length(), b.bit_length())
        return min(b, max(a, self.between(1 << (hi - 1), (1 << hi) - 1)))


def filler(seed, n):
    """n pseudo-random bytes (SHAKE-128 of the seed): cheap bulk content for uncompressed chunks."""
    return hashlib.shake_128(struct.pack("<Q", seed & M64)).digest(n)


# ---- range encoder and the LZMA model ----

class RangeEncoder:
    def __init__(self):
        self.low, self.range, self.cache, self.cache_size = 0, 0xFFFFFFFF, 0, 1
        self.out = bytearray()

    def _shift_low(self):
        if self.low < 0xFF000000 or self.low >= 1 << 32:
            carry = self.low >> 32
            temp = self.cache
            while True:
                self.out.append((temp + carry) & 0xFF)
                temp = 0xFF
                self.cache_size -= 1
                if self.cache_size == 0:
                    break
            self.cache = (self.low >> 24) & 0xFF
        self.cache_size += 1
        self.low = (self.low & 0x00FFFFFF) << 8

    def bit(self, p, i, b):
        prob = p[i]
        bound = (self.range >> 11) * prob
        if b:
            self.low += bound
            self.range -= bound
            p[i] = prob - (prob >> 5)
        else:
            self.range = bound
            p[i] = prob + ((2048 - prob) >> 5)
        while self.range < 1 << 24:
            self.range <<= 8
            self._shift_low()

    def direct(self, v, nbits):
        for i in range(nbits - 1, -1, -1):
            self.range >>= 1
            if (v >> i) & 1:
                self.low += self.range
            while self.range < 1 << 24:
                self.range <<= 8
                self._shift_low()

    def tree(self, p, base, nbits, sym):
        m = 1
        for i in range(nbits - 1, -1, -1):
            b = (sym >> i) & 1
            self.bit(p, base + m, b)
            m = (m << 1) | b

    def rtree(self, p, base, nbits, sym):
        m = 1
        for _ in range(nbits):
            b = sym & 1
            sym >>= 1
            self.bit(p, base + m, b)
            m = (m << 1) | b

    def size_bound(self):
        """Bytes the chunk has if it is flushed now."""
        return len(self.out) + self.cache_size + 4

    def finish(self):
        for _ in range(5):
            self._shift_low()
        return bytes(self.out)


# offsets into one flat probability list
IS_MATCH, IS_REP, IS_REP0, IS_REP1, IS_REP2, IS_REP0_LONG = 0, 192, 204, 216, 228, 240
DIST_SLOT, POS_SPECIAL, ALIGN = 432, 688, 802
MATCH_LEN, REP_LEN = 818, 1332          # choice, choice2, low[16][8], mid[16][8], high[256]
LITERAL = 1846


def dist_slot(d):
    if d < 4:
        return d
    n = d.bit_length() - 1
    return 2 * n + ((d >> (n - 1)) & 1)


def slot_range(slot):
    """The distances (rep0 values) slot codes: [lo, hi]."""
    if slot < 4:
        return slot, slot
    n = (slot >> 1) - 1
    lo = (2 | (slot & 1)) << n
    return lo, lo + (1 << n) - 1


def dict_size_of(prop):
    return 0xFFFFFFFF if prop == 40 else (2 | (prop & 1)) << (prop // 2 + 11)


class Coverage:
    def __init__(self):
        self.state_kind = set()
        self.slots = set()                  # (len_to_pos_state, slot)
        self.match_lens, self.rep_lens = set(), set()
        self.transitions = set()            # (previous control byte or None, control byte); 0x00 = end marker
        self.lzma_start_mod16, self.reset_mod16 = set(), set()
        self.props = set()
        self.events = collections.Counter()


def valid_transitions():
    """Every (previous control, control) pair that some valid LZMA2 stream contains (lzma2_decoder.c's rules; whether
    0x80 / 0xA0 may follow 0x02 also depends on the chunks before it, see Block.need_props)."""
    out = {(None, 0x00), (None, 0x01), (None, 0xE0)}
    for prev in (0x01, 0x02) + LZMA_CTRL:
        for c in (0x00, 0x01, 0x02, 0xC0, 0xE0):
            out.add((prev, c))
        if prev != 0x01:   # 0x01 leaves the properties unset until the next 0xC0 / 0xE0
            out |= {(prev, 0x80), (prev, 0xA0)}
    return out


# pending-copy geometry of the warp decoder (xzb_dec_warp.cuh), mirrored to count which forms the symbols reach
GEOMETRY_EVENTS = ("mb_in_pending", "mb_at_pending_start", "src_in_pending", "short_rep_after_pending", "pending_at_chunk_end",
                   "pending_then_dict_reset", "period<32_len<=32", "period<32_len>32", "period=32_len<=32", "period=32_len>32",
                   "period>32_len<=32", "period>32_len>32")
WINDOW_EVENTS = ("dist_full-1_dict_full", "dist_full-1_after_reset", "lit_prev0_after_reset", "lit_prev_from_uncompressed",
                 "lit_equals_match_byte", "len2_far")


class Block:
    """One Block's LZMA2 payload and plaintext, built chunk by chunk."""

    def __init__(self, seed, dict_prop, cov):
        self.rng = Rng(seed)
        self.seed = seed
        self.dict_prop = dict_prop
        self.dict_size = dict_size_of(dict_prop)
        d = max(self.dict_size, 4096)
        self.dict_r = 0xFFFFFFF0 if d > 0xFFFFFFF0 else (d + 15) & ~15
        self.cov = cov
        self.out, self.payload = bytearray(), bytearray()
        self.dict_start = 0
        self.prev_ctrl = None
        self.need_props = True
        self.declared = 0
        self.props = None
        self.p = None
        self.state = 0
        self.reps = [0, 0, 0, 0]
        self.pend = None        # (start, length) of the warp decoder's deferred copy
        self.nchunk = 0
        self.first_after_u = False

    # ---- chunk level ----
    def _control(self, ctrl, near_miss=False):
        if not near_miss:
            assert (self.prev_ctrl, ctrl) in valid_transitions(), (self.prev_ctrl, ctrl)
            assert not (self.need_props and ctrl in (0x80, 0xA0)), "0x80 / 0xA0 before any 0xC0 / 0xE0 after an 0x01"
        if self.pend is not None and ctrl != 0x00:   # the deferred copy was stored at the end of the previous chunk
            if ctrl in (0x01, 0xE0):
                self.cov.events["pending_then_dict_reset"] += 1
        self.pend = None
        if not near_miss:
            self.cov.transitions.add((self.prev_ctrl, ctrl))
        self.prev_ctrl = ctrl
        if ctrl in (0x01, 0xE0):
            if self.out:
                self.cov.reset_mod16.add(len(self.out) % 16)
            self.dict_start = len(self.out)
        if ctrl == 0x01:
            self.need_props = True
        elif ctrl >= 0xC0:
            self.need_props = False

    def uncompressed(self, n, reset=False, data=None):
        assert 1 <= n <= 65536
        self._control(0x01 if reset else 0x02)
        data = filler(self.seed * 1000003 + self.nchunk, n) if data is None else data
        self.nchunk += 1
        self.payload += bytes([0x01 if reset else 0x02, (n - 1) >> 8, (n - 1) & 0xFF]) + data
        self.out += data
        self.declared += n

    def lzma(self, ctrl, target, mix, props=None, script=None, valid=True):
        """One LZMA chunk of up to `target` bytes (fewer if 64 KiB of compressed bytes come first); returns its size.
        script(block, rc), when given, codes the symbols instead and returns the Uncompressed Size to declare (None: the
        bytes it produced)."""
        after_u = self.prev_ctrl in (0x01, 0x02)
        self._control(ctrl, not valid)
        self.nchunk += 1
        if ctrl >= 0xC0:
            self.props = props
            self.p = [1024] * (LITERAL + (0x300 << (props[0] + props[1])))
        if ctrl >= 0xA0:
            self.p = [1024] * len(self.p)
            self.state, self.reps = 0, [0, 0, 0, 0]
        if valid:
            self.cov.props.add(self.props)
        start = len(self.out)
        self.cov.lzma_start_mod16.add(start % 16)
        self.first_after_u = after_u
        rc = RangeEncoder()
        declared = None
        if script is not None:
            declared = script(self, rc)
        else:
            while len(self.out) - start < target and rc.size_bound() + 64 <= 65536:
                self._symbol(rc, target - (len(self.out) - start), mix)
        usize = len(self.out) - start if declared is None else declared
        if self.pend is not None:
            self.cov.events["pending_at_chunk_end"] += 1
        data = rc.finish()
        assert 1 <= usize <= 2 * MiB and len(data) <= 65536
        hdr = bytes([ctrl | ((usize - 1) >> 16), ((usize - 1) >> 8) & 0xFF, (usize - 1) & 0xFF, (len(data) - 1) >> 8, (len(data) - 1) & 0xFF])
        if ctrl >= 0xC0:
            lc, lp, pb = self.props
            hdr += bytes([(pb * 5 + lp) * 9 + lc])
        self.payload += hdr + data
        self.declared += usize
        return usize

    def end(self):
        self._control(0x00)
        self.payload.append(0x00)

    # ---- symbol level ----
    def full(self):
        rel = len(self.out) - self.dict_start
        return rel if rel < self.dict_r else self.dict_r

    def _symbol(self, rc, rem, mix):
        rng, full, reps = self.rng, self.full(), self.reps
        kinds = [("lit", mix.w.get("lit", 0))]
        if full > 0 and rem >= 2:
            kinds.append(("match", mix.w.get("match", 0)))
        if full > reps[0]:
            kinds.append(("short", mix.w.get("short", 0)))
        if rem >= 2:
            kinds += [("rep%d" % i, mix.w.get("rep", 0)) for i in range(4) if full > reps[i]]
        kinds = [(k, w) for k, w in kinds if w] or [("lit", 1)]
        kind = rng.pick(kinds)
        if kind == "lit":
            self.literal(rc, None, mix)
        elif kind == "short":
            self.short_rep(rc)
        elif kind == "match":
            dist = self._distance(full, mix)
            self.match(rc, dist, self._length(min(273, rem), dist, mix))
        else:
            i = int(kind[3])
            self.rep(rc, i, self._length(min(273, rem), reps[i], mix))

    def _distance(self, full, mix):
        rng = self.rng
        mode = rng.pick(mix.dist)
        if mode == "near":
            return rng.between(0, min(40, full - 1))
        if mode == "edge":
            return max(0, full - 1 - (0 if rng.below(2) else rng.between(0, 3)))
        lo, hi = slot_range(rng.between(0, dist_slot(full - 1)))
        return rng.between(lo, min(hi, full - 1))

    def _length(self, top, dist, mix):
        rng = self.rng
        mode = rng.pick(mix.lens)
        if mode == "period" and 2 <= dist + 1 <= top:
            return dist + 1
        if mode == "short":
            return rng.between(2, min(top, 34))
        if mode == "long":
            return rng.between(max(2, top - 40), top)
        return rng.between(2, top)

    def _pos_state(self):
        return (len(self.out) - self.dict_start) & ((1 << self.props[2]) - 1)

    def _kind(self, kind):
        self.cov.state_kind.add((self.state, kind))
        self.first_after_u = False

    def literal(self, rc, byte, mix=None):
        rng, out, p = self.rng, self.out, self.p
        lc, lp, _ = self.props
        rel = len(out) - self.dict_start
        prev = out[-1] if rel > 0 else 0
        if rel == 0 and self.dict_start > 0:
            self.cov.events["lit_prev0_after_reset"] += 1
        if self.first_after_u and rel > 0:
            self.cov.events["lit_prev_from_uncompressed"] += 1
        ps = self._pos_state()
        self._kind("lit")
        rc.bit(p, IS_MATCH + self.state * 16 + ps, 0)
        base = LITERAL + 0x300 * (((rel & ((1 << lp) - 1)) << lc) + (prev >> (8 - lc)))
        full = self.full()
        if self.state >= 7 and full > self.reps[0]:
            mb = out[-self.reps[0] - 1]
            if self.pend is not None and len(out) - self.reps[0] - 1 >= self.pend[0]:
                self.cov.events["mb_in_pending"] += 1
                if len(out) - self.reps[0] - 1 == self.pend[0]:
                    self.cov.events["mb_at_pending_start"] += 1
            if byte is None:
                r = rng.below(8)
                byte = mb if r < mix.lit_eq else (mb ^ (1 << rng.below(8))) if r < 6 else rng.below(256)
            if byte == mb:
                self.cov.events["lit_equals_match_byte"] += 1
            offset, sym, m = 0x100, 1, mb
            for i in range(7, -1, -1):
                m <<= 1
                match_bit = m & offset
                b = (byte >> i) & 1
                rc.bit(p, base + offset + match_bit + sym, b)
                sym = (sym << 1) | b
                offset &= match_bit if b else ~match_bit
        else:
            if byte is None:
                byte = rng.below(256) if rng.below(4) else (prev + 1) & 0xFF
            rc.tree(p, base, 8, byte)
        self.state = 0 if self.state < 4 else self.state - 3 if self.state < 10 else self.state - 6
        out.append(byte)

    def _length_code(self, rc, base, length, ps, lens):
        lens.add(length)
        l = length - 2
        if l < 8:
            rc.bit(self.p, base, 0)
            rc.tree(self.p, base + 2 + ps * 8, 3, l)
        elif l < 16:
            rc.bit(self.p, base, 1)
            rc.bit(self.p, base + 1, 0)
            rc.tree(self.p, base + 130 + ps * 8, 3, l - 8)
        else:
            rc.bit(self.p, base, 1)
            rc.bit(self.p, base + 1, 1)
            rc.tree(self.p, base + 258, 8, l - 16)

    def match(self, rc, dist, length, apply=True, past_edge=False):
        p, ps = self.p, self._pos_state()
        self._kind("match")
        rc.bit(p, IS_MATCH + self.state * 16 + ps, 1)
        rc.bit(p, IS_REP + self.state, 0)
        self._length_code(rc, MATCH_LEN, length, ps, self.cov.match_lens)
        lps = min(length - 2, 3)
        slot = dist_slot(dist)
        self.cov.slots.add((lps, slot))
        rc.tree(p, DIST_SLOT + lps * 64, 6, slot)
        if slot >= 4:
            nbits = (slot >> 1) - 1
            reduced = dist - slot_range(slot)[0]
            if slot < 14:
                rc.rtree(p, POS_SPECIAL + slot_range(slot)[0] - slot - 1, nbits, reduced)
            else:
                rc.direct(reduced >> 4, nbits - 4)
                rc.rtree(p, ALIGN, 4, reduced & 15)
        if length == 2 and slot >= 14:
            self.cov.events["len2_far"] += 1
        self.state = 7 if self.state < 7 else 10
        self.reps = [dist] + self.reps[:3]
        if apply:
            self._copy(length, past_edge)

    def rep(self, rc, i, length, apply=True, past_edge=False):
        p, ps = self.p, self._pos_state()
        self._kind("rep%d" % i)
        rc.bit(p, IS_MATCH + self.state * 16 + ps, 1)
        rc.bit(p, IS_REP + self.state, 1)
        if i == 0:
            rc.bit(p, IS_REP0 + self.state, 0)
            rc.bit(p, IS_REP0_LONG + self.state * 16 + ps, 1)
        else:
            rc.bit(p, IS_REP0 + self.state, 1)
            if i == 1:
                rc.bit(p, IS_REP1 + self.state, 0)
            else:
                rc.bit(p, IS_REP1 + self.state, 1)
                rc.bit(p, IS_REP2 + self.state, 0 if i == 2 else 1)
        self.reps = [self.reps[i]] + [r for j, r in enumerate(self.reps) if j != i]
        self.state = 8 if self.state < 7 else 11
        self._length_code(rc, REP_LEN, length, ps, self.cov.rep_lens)
        if apply:
            self._copy(length, past_edge)

    def short_rep(self, rc, apply=True):
        p, ps = self.p, self._pos_state()
        self._kind("short")
        if self.pend is not None:
            self.cov.events["short_rep_after_pending"] += 1
        rc.bit(p, IS_MATCH + self.state * 16 + ps, 1)
        rc.bit(p, IS_REP + self.state, 1)
        rc.bit(p, IS_REP0 + self.state, 0)
        rc.bit(p, IS_REP0_LONG + self.state * 16 + ps, 0)
        self.state = 9 if self.state < 7 else 11
        if apply:
            self._copy(1)

    def _copy(self, length, past_edge=False):
        """Append the copy of the current match; past_edge: a near miss whose source lies just outside the window
        (the bytes are there, the decoder must refuse them)."""
        out, dist = self.out, self.reps[0]
        pos, full = len(out), self.full()
        assert (dist < full or past_edge and dist < pos) and length >= 1
        if dist == full - 1:
            if full == self.dict_r:
                self.cov.events["dist_full-1_dict_full"] += 1
            elif self.dict_start > 0:
                self.cov.events["dist_full-1_after_reset"] += 1
        period, back = dist + 1, pos - dist - 1
        ev = self.cov.events
        if self.pend is not None and back < self.pend[0] + self.pend[1] and back + length > self.pend[0]:
            ev["src_in_pending"] += 1
        ev["period%s32_len%s32" % ("<" if period < 32 else "=" if period == 32 else ">", "<=" if length <= 32 else ">")] += 1
        if period >= length:
            out += out[back:back + length]
        else:
            out += (out[back:] * (length // period + 1))[:length]
        self.pend = (pos, length) if length <= 32 else None


class Mix:
    def __init__(self, w, dist=(("slot", 1),), lens=(("any", 1),), lit_eq=2):
        self.w, self.dist, self.lens, self.lit_eq = dict(w), list(dist), list(lens), lit_eq


MIXES = {
    "literal": Mix({"lit": 12, "match": 2, "short": 1, "rep": 1}, lens=(("short", 3), ("any", 1))),
    "rep": Mix({"lit": 3, "match": 2, "short": 3, "rep": 3}, dist=(("near", 1), ("slot", 2)), lens=(("short", 2), ("any", 1))),
    "far": Mix({"lit": 2, "match": 6, "short": 1, "rep": 1}, dist=(("slot", 1),), lens=(("short", 2), ("any", 1), ("period", 0))),
    "overlap": Mix({"lit": 3, "match": 5, "short": 2, "rep": 2}, dist=(("near", 1),), lens=(("short", 3), ("any", 2), ("period", 2))),
    "edge": Mix({"lit": 2, "match": 4, "short": 1, "rep": 2}, dist=(("edge", 3), ("near", 1), ("slot", 1)), lens=(("short", 2), ("any", 1))),
    "long": Mix({"lit": 1, "match": 1, "rep": 30}, dist=(("near", 1),), lens=(("long", 1),)),
}


# ---- the .xz wrapper ----

def _vli(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _crc64_table():
    t = []
    for b in range(256):
        r = b
        for _ in range(8):
            r = (r >> 1) ^ (0xC96C5795D7870F42 if r & 1 else 0)
        t.append(r)
    return t


_CRC64 = _crc64_table()


def crc64(data):
    """CRC-64/XZ (ECMA-182 polynomial, reflected), bytewise: the generator uses it on Blocks of a few MiB at most."""
    c, t = M64, _CRC64
    for b in data:
        c = t[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ M64


def check_field(check, data):
    if check == 0:
        return b""
    if check == 1:
        return struct.pack("<I", zlib.crc32(data))
    if check == 4:
        return struct.pack("<Q", crc64(data))
    assert check == 10
    return hashlib.sha256(data).digest()


def xz_stream(payload, dict_prop, uncomp, check, data):
    """One Stream of one sized Block (LZMA2 only); the Check field is that of `data`."""
    flags = bytes([0, check])
    out = bytearray(b"\xfd7zXZ\x00" + flags + struct.pack("<I", zlib.crc32(flags)))
    body = bytes([0xC0]) + _vli(len(payload)) + _vli(uncomp) + b"\x21\x01" + bytes([dict_prop])
    body += b"\0" * (-(len(body) + 5) % 4)
    hdr = bytes([(len(body) + 5) // 4 - 1]) + body
    hdr += struct.pack("<I", zlib.crc32(hdr))
    cf = check_field(check, data)
    out += hdr + payload + b"\0" * (-len(payload) % 4) + cf
    idx = b"\0" + _vli(1) + _vli(len(hdr) + len(payload) + len(cf)) + _vli(uncomp)
    idx += b"\0" * (-len(idx) % 4)
    idx += struct.pack("<I", zlib.crc32(idx))
    tail = struct.pack("<I", len(idx) // 4 - 1) + flags
    return bytes(out + idx + struct.pack("<I", zlib.crc32(tail)) + tail + b"YZ")


Case = collections.namedtuple("Case", "name payload dict_size expected verdict xz declared check")


def _case(name, b, check, verdict=0):
    data = bytes(b.out)
    if verdict == 0:
        assert b.declared == len(data)
    return Case(name, bytes(b.payload), b.dict_size, data, verdict, xz_stream(bytes(b.payload), b.dict_prop, b.declared, check, data),
                b.declared, check)


def uncompressed_payload(data):
    """An LZMA2 payload of uncompressed chunks only (0x01, then 0x02) that decodes to data."""
    out = bytearray()
    for i in range(0, len(data), 65536):
        part = data[i:i + 65536]
        out += bytes([0x01 if i == 0 else 0x02, (len(part) - 1) >> 8, (len(part) - 1) & 0xFF]) + part
    out.append(0x00)
    return bytes(out)


# ---- case families ----

CHECKS = (0, 1, 4, 10)


def _symbol_mix(cov):
    cases = []
    for k, mix in enumerate(("literal", "rep", "far", "overlap")):
        for s in range(3):
            seed = 100 + 10 * k + s
            props = PROPS[(7 * seed) % len(PROPS)]
            b = Block(seed, 20 + s, cov)            # dictionaries of 1, 1.5 and 2 MiB
            rng = b.rng
            b.lzma(0xE0, rng.between(1, 300), MIXES["literal"], props)   # something to match against
            for _ in range(3 + s):
                b.lzma(rng.pick([(0x80, 3), (0xA0, 1)]), rng.between(20000, 120000), MIXES[mix])
            b.end()
            cases.append(_case("mix_%s_%d" % (mix, s), b, CHECKS[(k + s) % 4]))
    return cases


def _churn(cov):
    cases = []
    valid = valid_transitions()
    props_i = 0
    for s in range(6):
        seed = 200 + s
        b = Block(seed, 23, cov)                    # 12 MiB
        rng = b.rng
        nchunks = 50 + 10 * s
        for c in range(nchunks + 1):
            last = c == nchunks
            if last:
                ctrl = 0x00
            else:
                opts = [x for x in (0x01, 0x02) + LZMA_CTRL if (b.prev_ctrl, x) in valid and not (b.need_props and x in (0x80, 0xA0))]
                fresh = [x for x in opts if (b.prev_ctrl, x) not in cov.transitions]
                if c == nchunks - 1:     # end the Block after a control byte the earlier Blocks did not end after
                    fresh = [x for x in opts if (x, 0x00) not in cov.transitions] or fresh
                ctrl = fresh[rng.below(len(fresh))] if fresh and rng.below(3) else opts[rng.below(len(opts))]
            if ctrl == 0x00:
                break
            if ctrl in (0x01, 0x02):
                n = rng.pick([(1, 1), (65536, 1), (rng.log_between(1, 65536), 6)])
                b.uncompressed(n, ctrl == 0x01)
                continue
            props = None
            if ctrl >= 0xC0:
                props = PROPS[props_i % len(PROPS)]
                props_i += 1
            if c == 7 and s < 2:
                b.lzma(ctrl, 2 * MiB, MIXES["long"], props)    # exactly 2 MiB unpacked
                continue
            target = rng.pick([(1, 1), (rng.between(2, 16), 2), (rng.log_between(17, 30000), 6)])
            b.lzma(ctrl, target, MIXES[rng.pick([("literal", 1), ("rep", 1), ("overlap", 2), ("far", 1)])], props)
        b.end()
        cases.append(_case("churn_%d" % s, b, CHECKS[s % 4]))
    return cases


def _window_edge(cov):
    cases = []
    for s, (prop, size) in enumerate(((0, 40 << 10), (1, 100 << 10), (2, 200 << 10), (0, 150 << 10), (1, 64 << 10), (2, 120 << 10))):
        seed = 300 + s
        b = Block(seed, prop, cov)
        rng = b.rng
        props = PROPS[(13 * seed) % len(PROPS)]
        b.lzma(0xE0, rng.between(1, 5000), MIXES["literal"], props)
        while b.declared < size:
            r = rng.below(8)
            if r == 0:        # a dictionary reset in the middle of the Block: 0xE0, or 0x01 then 0xC0
                b.lzma(0xE0, rng.between(1, 20000), MIXES["edge"], PROPS[rng.below(len(PROPS))])
            elif r == 1:
                b.uncompressed(rng.between(1, 3000), True)
                b.lzma(0xC0, rng.between(1, 20000), MIXES["edge"], PROPS[rng.below(len(PROPS))])
            elif r == 2:
                b.uncompressed(rng.between(1, 3000))
            else:
                b.lzma(0x80, rng.between(1000, 30000), MIXES["edge"])
        b.end()
        cases.append(_case("window_%d_%d" % (dict_size_of(prop), s), b, CHECKS[s % 4]))
    return cases


def _big(cov):
    """About 80 MiB: uncompressed chunks, then far matches up to the largest distance the Block allows."""
    b = Block(400, 29, cov)                         # 96 MiB dictionary, so `full` is the Block's size
    rng = b.rng
    b.uncompressed(65536, True)
    while b.declared < 78 * MiB:
        b.uncompressed(65536)
    b.lzma(0xC0, 2 * MiB, MIXES["far"], (3, 0, 2))

    def farthest(b, rc):        # the last chunk ends on the farthest matches the Block allows
        b.literal(rc, None, MIXES["far"])
        b.match(rc, b.full() - 1, 2)
        b.match(rc, b.full() - 1, 273)
    b.lzma(0x80, 0, None, script=farthest)
    b.end()
    return [_case("big", b, 1)]


def _high_ratio(cov):
    b = Block(500, 26, cov)                         # 32 MiB
    b.lzma(0xE0, 64, MIXES["literal"], (0, 0, 0))
    while b.declared < 16 * MiB:
        b.lzma(0x80, 2 * MiB, MIXES["long"])
    b.end()
    return [_case("high_ratio", b, 1)]


def _empty(cov):
    b = Block(600, 0, cov)
    b.end()
    return [_case("empty", b, 1)]


def _near_misses(cov):
    """One symbol or control byte past an edge, the rest valid: the decoders must say LZMA_DATA_ERROR.  A decoder one
    step off at the edge would accept the symbol (its source bytes are in the buffer) and decode the rest."""
    cases = []
    lit = MIXES["literal"]

    def rest(b, rc):
        for _ in range(300):
            b._symbol(rc, 100000, MIXES["overlap"])

    def dist_full(b, rc):                       # rep0 == full (4096, the dictionary) in a Block longer than it
        b.literal(rc, None, lit)
        b.match(rc, b.full(), 5, past_edge=True)
        rest(b, rc)

    def past_chunk(b, rc):                      # a match longer than what is left of the chunk
        for _ in range(40):
            b.literal(rc, None, lit)
        b.match(rc, 3, 20, apply=False)
        return 50

    def rep_at_reset(b, rc):                    # a rep right after a mid-Block dictionary reset: full == 0
        b.rep(rc, 0, 4, past_edge=True)
        rest(b, rc)

    for name, ctrl, fn in (("dist_eq_full", 0x80, dist_full), ("match_past_chunk", 0x80, past_chunk), ("rep_after_reset", 0xE0, rep_at_reset)):
        b = Block(700 + len(cases), 0, cov)
        b.lzma(0xE0, 5000, MIXES["overlap"], (3, 0, 2))
        b.lzma(ctrl, 0, None, (1, 1, 1), script=fn, valid=False)
        b.end()
        cases.append(_case("nearmiss_" + name, b, 1, DATA_ERROR))
    # 0x80 right after 0x01
    b = Block(710, 0, cov)
    b.lzma(0xE0, 2000, MIXES["overlap"], (3, 0, 2))
    b.uncompressed(100, True)
    b.lzma(0x80, 0, None, script=lambda b, rc: (b.literal(rc, None, lit), 1)[1], valid=False)
    b.end()
    cases.append(_case("nearmiss_0x80_after_0x01", b, 1, DATA_ERROR))
    # lc + lp > 4 in a 0xC0 in the middle of the Block
    b = Block(711, 0, cov)
    b.lzma(0xE0, 2000, MIXES["overlap"], (3, 0, 2))
    b._control(0xC0, near_miss=True)
    b.payload += bytes([0xC0, 0, 9, 0, 4, (0 * 5 + 2) * 9 + 3]) + bytes([0, 0x10, 0x20, 0x30, 0x40])
    b.declared += 10
    b.end()
    cases.append(_case("nearmiss_lclp_gt4", b, 1, DATA_ERROR))
    return cases


_cached = {}


def cases():
    """All cases, generated once per process."""
    if "cases" not in _cached:
        cov = Coverage()
        out = []
        for fam in (_symbol_mix, _churn, _window_edge, _big, _high_ratio, _empty, _near_misses):
            out += fam(cov)
        _cached["cases"], _cached["cov"] = out, cov
    return _cached["cases"]


def coverage():
    cases()
    return _cached["cov"]
