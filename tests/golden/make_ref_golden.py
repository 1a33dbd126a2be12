#!/usr/bin/env python
"""Regenerates tests/golden/ref_live_golden.json from the UNMODIFIED reference
(oracle/_ref, built by oracle/Makefile.ref where the reference tree exists).

The reference's answers on the tests' seeded inputs (filters, encoders, decoder verdicts, the <lzma.h>
struct layout, `xz -6 -T1` Streams, the LZMA2 option sweep of test_gpu_option_sweep.py and its Streams with rewritten
dictionary sizes, the decoder's verdicts on the Streams of tests/lzma2_gen.py, the Streams of the chunk-mix cases of
tests/chunk_mix.py), stored as the first 48 bits of SHA-256.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
import xzlibs as X
import test_api_cpu as API
import test_filters_cpu as F
import test_gpu_filters as G
import test_gpu_option_sweep as S
import test_oracle as O
import lzma2_gen
import chunk_mix

sys.path.insert(0, os.path.dirname(TESTS))
REF = __import__("__graft_entry__").reference_tree()   # the reference source tree (for its public header)


sha = X.sha64


def ref_apply(fid, arg, enc, data):
    n = len(data)
    out = (C.c_uint8 * max(n, 1))()
    ids = (C.c_uint32 * 1)(fid); args = (C.c_uint32 * 1)(arg)
    r = X.ref().ref_filter_apply(ids, args, C.c_uint32(1), C.c_int(enc), bytes(data), C.c_size_t(n), out)
    assert r == 0, r
    return bytes(out[:n])


def ref_chain_encode(data, chain, preset, bs, check=4):
    n = len(data)
    cap = n + n // 2 + 65536
    out = (C.c_uint8 * cap)()
    sz = C.c_size_t()
    ids = (C.c_uint32 * len(chain))(*[c[0] for c in chain])
    args = (C.c_uint32 * len(chain))(*[c[1] for c in chain])
    r = X.ref().ref_encode_mt_chain(data, C.c_size_t(n), ids, args, C.c_uint32(len(chain)), C.c_uint32(preset), C.c_uint64(bs), C.c_uint32(check),
                                    C.c_uint32(4), out, C.c_size_t(cap), C.byref(sz))
    assert r == 0, r
    return bytes(out[:sz.value])


def opt_sweep():
    """lzma_stream_encoder_mt with each sweep case's LZMA2 options."""
    out = {}
    for c in S.sweep_cases():
        threads = 1 if c.opts.dict_size >= 64 * S.MiB else 0   # about 0.6 GiB of match finder per thread at 64 MiB
        out[S.key(c)] = sha(X.ref_encode(c.data, len(c.data), 0, c.block_size, c.check, threads=threads, opts=c.opts))
    return out


def dict_header():
    """The single-threaded decoder's [ret, out_size, output] on Streams whose Block Headers announce each dictionary
    size property (and invalid ones)."""
    out = {}
    for name, o, bs, data in S.dict_header_streams():
        xz = X.ref_encode(data, len(data), 0, bs, opts=o)
        props = {}
        for prop in S.DICT_PROPS:
            r, back = X.ref_decode(S.set_dict_prop(xz, prop), len(data))
            props[str(prop)] = [r, len(back), sha(back)]
        out[name] = {"stream": sha(xz), "props": props}
    return out


def lzma2_gen_section():
    """The single-threaded and threaded decoders' [ret, out_size, output] on each generated Stream, and the
    single-threaded decoder's on the same Stream without the Block Header's size fields.  A valid case's output must be
    the generator's plaintext: a generator bug is not recorded as the reference's answer."""
    out = {}
    for c in lzma2_gen.cases():
        unsized = X.drop_block_sizes(c.xz)
        res = [X.ref_decode(c.xz, c.declared), X.ref_decode(c.xz, c.declared, mt=True), X.ref_decode(unsized, c.declared)]
        for r, back in res:
            if c.verdict == 0:
                assert r == 0 and back == c.expected, (c.name, r, len(back))
            else:
                assert r == c.verdict, (c.name, r)
        out[c.name] = {"stream": sha(c.xz), "decode": [[r, len(back), sha(back)] for r, back in res]}
    return out


def chunk_mix_section():
    """lzma_stream_encoder_mt with each chunk-mix case's options ([LZMA chunks, uncompressed chunks] read from its
    Blocks), and lzma_easy_buffer_encode of each one-shot item.  The oracle must write the same Stream: a difference is
    an oracle bug, not an answer to record."""
    out = {}
    for c in chunk_mix.cases():
        xz = X.ref_encode(c.data, len(c.data), 0, c.block_size, c.check, opts=c.opts)
        assert X.oracle_encode(c.data, len(c.data), 0, c.block_size, c.check, opts=c.opts) == xz, c.name
        out[chunk_mix.key(c)] = {"stream": sha(xz), "chunks": list(chunk_mix.chunk_counts(xz))}
    for name, p, data in chunk_mix.oneshot_items():
        xz = X.ref_buffer_encode(data, len(data), p)
        assert X.oracle_buffer_encode(data, len(data), p) == xz, name
        out[name] = {"stream": sha(xz)}
    return out


def main():
    assert X.have_ref(), "oracle/_ref is not built"
    assert REF and os.path.isdir(REF), "the reference source tree is not there (XZ_REFERENCE)"
    g = {"filter_apply": {}, "chain_encode": {}, "buffer_encode": {}, "buffer_decode": {}, "stream_encode": {}, "stream_decode": {},
         "mf_encode": {}}
    cases = [(fid, arg, n, F.codeish(fid, n, 1000 * fid + n)) for fid, arg, n in F.BCJ_CASES]
    cases += [(3, dist, n, F.delta_input(dist, n)) for dist, n in F.DELTA_CASES]
    for fid, arg, n, data in cases:
        g["filter_apply"].setdefault(f"{fid}|{arg}", {})[str(n)] = [sha(ref_apply(fid, arg, enc, data)) for enc in (1, 0)]
    for chain, preset, n, bs, data in G.chain_cases():
        g["chain_encode"][G.key(chain, preset, n, bs)] = sha(ref_chain_encode(data, chain, preset, bs))
    for kind, preset, n, check in O.BUFFER_CASES + [("E", 2, 3 * (1 << 20) + 17, 4)]:
        buf = X.gendata(kind, n)
        xz = X.ref_buffer_encode(buf, n, preset, check)
        k = O.key(kind, preset, n, check)
        g["buffer_encode"][k] = sha(xz)
        r, back, used = X.ref_buffer_decode(xz, n)
        g["buffer_decode"][k] = [r, used == len(xz), sha(back)]
    for kind in "TER":
        for preset, n, bs in O.STREAM_CASES:
            buf = X.gendata(kind, n)
            xz = X.ref_encode(buf, n, preset, bs)
            k = O.key(kind, preset, n, bs)
            g["stream_encode"][k] = sha(xz)
            g["stream_decode"][k] = [[r, sha(out)] for r, out in (X.ref_decode(xz, n), X.ref_decode(xz, n, mt=True))]
    buf = X.gendata("T", 300000)
    for o in O.mf_options():
        g["mf_encode"][O.mf_key(o)] = sha(X.ref_encode(buf, 300000, 0, 1 << 20, opts=o))
    g["opt_sweep"] = opt_sweep()
    g["dict_header"] = dict_header()
    g["lzma2_gen"] = lzma2_gen_section()
    g["chunk_mix"] = chunk_mix_section()
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "l.c")
        open(src, "w").write(API.LAYOUT_PROG.replace("HEADER", "<lzma.h>"))
        subprocess.check_call(["gcc", "-I", os.path.join(REF, "src", "liblzma", "api"), src, "-o", os.path.join(d, "l")])
        g["struct_layout"] = subprocess.check_output([os.path.join(d, "l")], text=True)
    # xz -6 -T1 Streams (single-threaded encoder: Blocks without Compressed / Uncompressed Size fields)
    xz = os.path.join(X.ROOT, "oracle", "_ref", "xz")
    g["xz_t1"] = {name: sha(subprocess.run([xz, "-6", "-T1"], input=data, stdout=subprocess.PIPE, check=True).stdout)
                  for name, data in (("T_300000", bytes(X.gendata("T", 300000)[:300000])), ("zeros_40000000", bytes(40 * 1000 * 1000)))}
    with open(os.path.join(HERE, "ref_live_golden.json"), "w") as f:   # one line per section
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(v, sort_keys=True, separators=(",", ":")) for k, v in sorted(g.items())) + "\n}\n")


if __name__ == "__main__":
    main()
