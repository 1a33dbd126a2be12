"""CPU tests of the device Stream decoder's logic (xz_b200/csrc/xzb_dec_stream.cuh): tests/hostsim/dec_stream_host.cpp runs
the round loop of xzb_stream_buffer_decode_batch_device -- scan, decode, filters, checks, settle, Index and Footer --
with the host forms of the decoder, the filters, CRC and SHA-256, so the same step functions the kernels run are checked
here against the reference's recorded results:
  * every file of the reference's decoder corpus gives its recorded verdict, and its bytes when it decodes;
  * the recorded lzma_stream_buffer_decode cases give their recorded ret, and in_used, size and hash of the output;
  * a batch of sized Streams and Streams whose Blocks carry no sizes walks in several rounds to the same results, also
    when a round holds only a few Blocks;
  * the grouping keeps every group within its budget and every item in exactly one group, in call order."""
import ctypes as C
import hashlib
import json
import os
import random
import sys

import pytest

import xzlibs as X

GOLD = os.path.join(X.ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
DATA_ERROR = 9
BUF_ERROR = 10


@pytest.fixture(scope="module")
def hs():
    lib = C.CDLL(os.path.join(X.ROOT, "tests", "hostsim", "libdecstreamhost.so"))
    lib.ds_plan_dec_groups.restype = C.c_uint32
    lib.ds_decode_batch.restype = C.c_int
    return lib


def decode(hs, streams, caps, flags=0, cap_jobs=65536, in_gap=0, out_gap=0):
    """[(ret, output bytes, in_used)] per Stream, and the rounds taken.  Items sit at odd offsets, in_gap / out_gap bytes
    apart; the bytes around every output slot must stay untouched."""
    n = len(streams)
    A = C.c_uint64 * max(n, 1)
    in_off, out_off = A(), A()
    pos, opos = 1, 3
    for i in range(n):
        in_off[i] = pos; pos += len(streams[i]) + in_gap
        out_off[i] = opos; opos += caps[i] + out_gap
    src = (C.c_uint8 * (pos + 1))()
    for i, s in enumerate(streams):
        C.memmove(C.addressof(src) + in_off[i], s, len(s))
    out = (C.c_uint8 * (opos + 1)).from_buffer(bytearray(b"\xa5" * (opos + 1)))
    size, used, rets, rounds = A(), A(), (C.c_uint32 * max(n, 1))(), C.c_uint32()
    r = hs.ds_decode_batch(C.c_uint32(n), src, in_off, A(*[len(s) for s in streams]), out, out_off, A(*caps), size, used, rets,
                           C.c_uint32(flags), C.c_uint32(cap_jobs), C.byref(rounds))
    assert r == 0
    raw = bytes(out)
    inside = bytearray(len(raw))
    for i in range(n):
        inside[out_off[i]: out_off[i] + caps[i]] = b"\x01" * caps[i]
    assert all(b == 0xA5 for b, m in zip(raw, inside) if not m), "a byte outside every slot changed"
    res = [(rets[i], raw[out_off[i]: out_off[i] + size[i]], used[i]) for i in range(n)]
    for i, (ret, _, _) in enumerate(res):
        if ret == 0:
            assert raw[out_off[i] + size[i]: out_off[i] + caps[i]] == b"\xa5" * (caps[i] - size[i])
    return res, rounds.value


def test_corpus_verdicts_and_bytes(hs):
    """Every file of the reference's decoder corpus, one batch: the recorded verdict (as the one-shot call maps it), size
    and hash, Delta / BCJ chains included."""
    verdicts = json.load(open(os.path.join(GOLD, "decode_verdicts.json")))
    names = sorted(verdicts)
    files = [open(os.path.join(GOLD, "ref_files", f), "rb").read() for f in names]
    got, _ = decode(hs, files, [1 << 20] * len(files))
    for name, (r, out, _) in zip(names, got):
        v = verdicts[name]
        want = DATA_ERROR if v["ret"] == BUF_ERROR else v["ret"]   # lzma_stream_buffer_decode's mapping of input that ends early
        assert r == want, (name, r, v["ret"])
        assert len(out) == v["out_size"], name
        if r == 0:
            assert hashlib.sha256(out).hexdigest() == v["out_sha256"], name
    assert len(names) > 50


def test_recorded_buffer_decode_cases(hs):
    """The recorded lzma_stream_buffer_decode cases, one batch per flags value: the reference's ret, and for ret == 0
    its in_used and output.  LZMA_CONCATENATED and the LZMA_TELL_* flags are the liblzma-named wrapper's, not this call's."""
    import make_golden as MG
    g = json.load(open(os.path.join(GOLD, "buffer_golden.json")))["decode"]
    enc, by_flags = {}, {}
    for name, kind, preset, n, m in MG.buffer_decode_cases():
        key = (kind, preset, n, m[0] == "nocheck")
        if key not in enc:
            enc[key] = X.oracle_buffer_encode(X.gendata(kind, n), n, preset, 0 if key[3] else 4)
        data, cap, flags = MG.buffer_apply(enc[key], n, m)
        if (flags & ~0x30) == 0:
            by_flags.setdefault(flags, []).append((name, data, cap))
    checked = 0
    for flags, group in sorted(by_flags.items()):
        got, _ = decode(hs, [d for _, d, _ in group], [c for _, _, c in group], 2 if flags & 0x10 else 0)
        for (name, _, _), (r, out, used) in zip(group, got):
            want = g[name]
            assert r == want["ret"], name
            if r == 0:
                assert (used, len(out), hashlib.sha256(out).hexdigest()) == (want["in_used"], want["out_size"], want["out_sha256"]), name
            checked += 1
    assert checked == 92   # flags 0, LZMA_IGNORE_CHECK and LZMA_FAIL_FAST


def _mixed_streams(count=30):
    """Sized multi-Block Streams, the same with their Block sizes dropped (one round per Block), one-shot Streams with
    and without sizes, all four checks, and empty items."""
    rng = random.Random(3)
    streams, items = [], []
    for i in range(count):
        n = rng.choice((0, 1, 4097, 70000, 200001))
        x = bytes(X.gendata("TER"[i % 3], n)[:n])
        check = (0, 1, 4, 10)[i % 4]
        if i % 4 == 0:
            s = X.oracle_encode(x, n, 1, 1 << 15, check=check)
        elif i % 4 == 1:
            s = X.drop_block_sizes(X.oracle_encode(x, n, 1, 1 << 15, check=check)) if n else X.oracle_buffer_encode(x, n, 1, check)
        elif i % 4 == 2:
            s = X.drop_block_sizes(X.oracle_buffer_encode(x, n, 1, check)) if n else X.oracle_buffer_encode(x, n, 1, check)
        else:
            s = X.oracle_buffer_encode(x, n, 3, check)
        streams.append(s); items.append(x)
    streams.append(b""); items.append(None)
    return streams, items


@pytest.mark.parametrize("cap_jobs", [65536, 5, 1])
def test_mixed_batch_walks_in_rounds(hs, cap_jobs):
    streams, items = _mixed_streams()
    caps = [len(x) if x is not None else 0 for x in items]
    got, rounds = decode(hs, streams, caps, cap_jobs=cap_jobs, in_gap=3, out_gap=0)
    for s, x, res in zip(streams, items, got):
        if x is None:
            assert res == (DATA_ERROR, b"", 0)
        else:
            assert res == (0, x, len(s))
    blocks = [0 if not x else -(-len(x) // (1 << 15)) if i % 4 < 2 else 1 for i, x in enumerate(items)]
    assert rounds >= max(b for i, b in enumerate(blocks) if i % 4 == 1) > 1   # an unsized Block takes a round of its own
    if cap_jobs == 1:
        assert rounds >= sum(blocks)


def test_short_slot_truncated_and_corrupt_items_in_one_batch(hs):
    """A slot one byte short, a cut Stream, a flipped byte in a Check field and a good neighbour: each its own verdict."""
    n = 150000
    x = bytes(X.gendata("T", n)[:n])
    s = X.oracle_encode(x, n, 1, 1 << 16, check=1)
    bad = bytearray(s); bad[-40] ^= 1
    got, _ = decode(hs, [s, s, s[:-30], bytes(bad), s], [n - 1, n, n, n, n + 9])
    assert got[0][0] == BUF_ERROR and got[1] == (0, x, len(s)) and got[2][0] == DATA_ERROR and got[4] == (0, x, len(s))
    assert got[3][0] == DATA_ERROR
    assert got[0][1] == x[:len(got[0][1])] and got[2][1] == x[:len(got[2][1])]


def test_grouping_keeps_budget_and_order(hs):
    rng = random.Random(9)
    sizes = [rng.choice((0, 1, 15, 16, 4096, 1 << 20, 40 << 20)) + rng.randrange(64) for _ in range(2000)]
    n = len(sizes)
    for per_item, budget in ((176, 1 << 30), (176, 64 << 20), (1000, 10 << 20), (176, 1)):
        group = (C.c_uint32 * n)()
        ng = hs.ds_plan_dec_groups((C.c_uint64 * n)(*sizes), C.c_uint32(n), C.c_uint64(per_item), C.c_uint64(budget), group)
        g = list(group)
        assert g[0] == 0 and g[-1] == ng - 1 and all(b - a in (0, 1) for a, b in zip(g, g[1:]))
        for k in range(ng):
            members = [i for i in range(n) if g[i] == k]
            cost = sum(per_item + 16 * (sizes[i] // 16 + 1) for i in members)
            assert members and (len(members) == 1 or cost <= budget)
    assert hs.ds_plan_dec_groups((C.c_uint64 * 1)(), C.c_uint32(0), C.c_uint64(1), C.c_uint64(1), (C.c_uint32 * 1)()) == 0
