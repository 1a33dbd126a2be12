// tests/hostsim/hostsim.cpp -- DEBUG HARNESS (tests only): compiles the product's host/device
// encoder and decoder logic (xz_b200/csrc/*.cuh) with g++ and runs it single-threaded so the
// logic can be checked against the oracle on a box without a GPU.  The CUDA-only plumbing
// (radix sort, kernel launch, work queues) is emulated with std::stable_sort and loops.
// Not part of the product and never used as a fallback.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../xz_b200/csrc/xzb_common.cuh"
#include "../../xz_b200/csrc/xzb_mf.cuh"
#include "xzb_enc.cuh"
#include "../../xz_b200/csrc/xzb_frame.cuh"
#include "../../xz_b200/csrc/xzb_params.h"
#include "../../xz_b200/csrc/xzb_dec.cuh"
#include "../../xz_b200/csrc/xzb_sha256.cuh"
#include "../../xz_b200/csrc/xzb_filters.cuh"

static XzbHostTables g_tab;
static bool g_tab_init = false;
static void tabs() { if (!g_tab_init) { xzb_make_tables(&g_tab); g_tab_init = true; } }

struct MfWork {
	std::vector<uint32_t> prev2, prev3, prevm, son, mh;
	std::vector<xzb_pair> mp, ovf;
	uint32_t ovf_top = 0, err = 0;
};

static void prev_by_key(const std::vector<uint32_t> &keys, uint32_t n_ins, std::vector<uint32_t> &prev, std::vector<uint32_t> *order_out)
{
	std::vector<uint32_t> order(n_ins);
	for (uint32_t i = 0; i < n_ins; ++i) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
	for (uint32_t i = 0; i < n_ins; ++i)
		prev[order[i]] = (i > 0 && keys[order[i - 1]] == keys[order[i]]) ? order[i - 1] : XZB_NONE;
	if (order_out) *order_out = order;
}

static void run_mf(const uint8_t *in, uint32_t n, const XzbParams &P, MfWork &W)
{
	W.prev2.assign(n, XZB_NONE); W.prev3.assign(n, XZB_NONE); W.prevm.assign(n, XZB_NONE);
	W.son.assign((size_t)2 * n + 2, 0xDEADBEEF);
	W.mh.assign(n, 0); W.mp.assign((size_t)n * P.mstride, xzb_pair{0, 0}); W.ovf.assign((size_t)n * 2 + 16, xzb_pair{0, 0});
	const uint32_t n_ins = n >= P.hash_bytes ? n - P.hash_bytes + 1 : 0;
	std::vector<uint32_t> k2(n_ins), k3(n_ins), km(n_ins), order;
	for (uint32_t p = 0; p < n_ins; ++p) { uint32_t h2 = 0, h3 = 0; km[p] = xzb_hash(in + p, P, g_tab.crc32, &h2, &h3); k2[p] = h2; k3[p] = h3; }
	if (P.hash_bytes >= 3) prev_by_key(k2, n_ins, W.prev2, nullptr);
	if (P.hash_bytes >= 4) prev_by_key(k3, n_ins, W.prev3, nullptr);
	prev_by_key(km, n_ins, W.prevm, &order);
	XzbMfBlock B;
	B.buf = in; B.n = n; B.room = n; B.prev2 = W.prev2.data(); B.prev3 = W.prev3.data(); B.prevm = W.prevm.data();
	B.son = W.son.data(); B.mh = W.mh.data(); B.mp = W.mp.data(); B.ovf = W.ovf.data();
	B.ovf_top = &W.ovf_top; B.ovf_cap = (uint32_t)W.ovf.size(); B.err = &W.err;
	if (!P.is_bt) {
		for (uint32_t p = 0; p < n; ++p) xzb_hc_position(B, P, p);
	} else {
		// bucket by bucket (any bucket order is valid; use sorted-key order like the GPU run list)
		for (uint32_t i = 0; i < n_ins; ++i) {
			const bool first = (i == 0) || km[order[i - 1]] != km[order[i]];
			xzb_bt_position(B, P, order[i], first ? XZB_NONE : order[i - 1]);
		}
		for (uint32_t p = n_ins; p < n; ++p) W.mh[p] = 0;
	}
}

extern "C" {

// Match store dump in the oracle's xzo_mf_dump layout (counts, longest, offsets, flat pairs).
uint64_t hs_mf_dump(const uint8_t *in, uint32_t n, const XzbLzmaOptions *opt, uint32_t *counts, uint32_t *longest,
		uint64_t *offsets, uint32_t *pairs, uint64_t pairs_cap)
{
	tabs();
	XzbParams P;
	if (xzb_make_params(opt, &P) != XZB_OK) return (uint64_t)-1;
	MfWork W;
	run_mf(in, n, P, W);
	if (W.err) return (uint64_t)-1;
	XzbMfView mf; mf.buf = in; mf.size = n; mf.read_pos = 0; mf.read_ahead = 0; mf.nice_len = P.nice_len; mf.stride = P.mstride;
	mf.mh = W.mh.data(); mf.mp = W.mp.data(); mf.ovf = W.ovf.data();
	uint64_t total = 0;
	xzb_pair m[XZB_MATCH_LEN_MAX + 1];
	for (uint32_t p = 0; p < n; ++p) {
		uint32_t c;
		const uint32_t lb = xzb_mfv_find(mf, &c, m);
		counts[p] = c; longest[p] = lb; offsets[p] = total;
		if (total + c > pairs_cap) return (uint64_t)-1;
		for (uint32_t i = 0; i < c; ++i) { pairs[2 * (total + i)] = m[i].len; pairs[2 * (total + i) + 1] = m[i].dist; }
		total += c;
	}
	return total;
}

int hs_block_encode(const uint8_t *in, uint32_t in_size, const XzbLzmaOptions *opt, uint32_t check, uint64_t block_size,
		uint8_t *out, uint32_t out_cap, XzbBlockResult *res)
{
	tabs();
	XzbParams P;
	int r = xzb_make_params(opt, &P);
	if (r != XZB_OK) return r;
	MfWork W;
	run_mf(in, in_size, P, W);
	if (W.err) return (int)W.err;
	XzbEnc *e = (XzbEnc *)malloc(sizeof(XzbEnc));
	xzb_enc_create(e, P, g_tab.prices);
	XzbMfView mf; mf.buf = in; mf.size = in_size; mf.read_pos = 0; mf.read_ahead = 0; mf.nice_len = P.nice_len; mf.stride = P.mstride;
	mf.mh = W.mh.data(); mf.mp = W.mp.data(); mf.ovf = W.ovf.data();
	// block_size == 0 selects the one-shot lzma_block_buffer_encode() framing
	const uint32_t oneshot = block_size == 0;
	uint64_t bound = xzbi_block_bound(block_size);
	uint32_t header_size = xzb_block_header_size(bound, block_size);
	if (oneshot) { header_size = xzb_block_header_size(xzb_lzma2_bound(in_size), in_size); bound = header_size + xzb_lzma2_bound(in_size); }
	uint32_t out_pos = header_size;
	r = xzb_lzma2_encode_block(e, mf, out, out_cap, &out_pos);
	uint64_t cv = 0;
	uint8_t cb[32] = { 0 };
	if (check == 1) cv = xzb_crc32_bytes(g_tab.crc32, in, in_size, 0);
	else if (check == 4) { uint64_t c = ~0ull; for (uint32_t i = 0; i < in_size; ++i) c = g_tab.crc64[(c ^ in[i]) & 0xFF] ^ (c >> 8); cv = ~c; }
	if (check == 10) xzb_sha256(in, in_size, cb); else for (int i = 0; i < 8; ++i) cb[i] = (uint8_t)(cv >> (8 * i));
	res->n_symbols = e->n_symbols; res->n_chunks_lzma = e->n_chunks_lzma; res->n_chunks_raw = e->n_chunks_raw;
	free(e);
	res->ret = XZB_OK;
	if (r == XZB_OK && xzb_block_finish_normal(g_tab.crc32, out, out_pos, header_size, bound, oneshot, check, cb, in_size, P.dict_prop, res)) return XZB_OK;
	xzb_block_finish_raw(g_tab.crc32, in, in_size, out, check, cb, res, 0, 1);
	return XZB_OK;
}

int hs_stream_encode(const uint8_t *in, uint64_t in_size, const XzbLzmaOptions *opt, uint32_t check, uint64_t block_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size)
{
	tabs();
	const uint64_t nblocks = (in_size + block_size - 1) / block_size;
	std::vector<uint64_t> unp(nblocks), unc(nblocks);
	uint64_t pos = xzb_stream_header(g_tab.crc32, out, check);
	const uint32_t cap = (uint32_t)(block_size + block_size / 4096 + 70000 + 1024);
	std::vector<uint8_t> scratch(cap);
	for (uint64_t b = 0; b < nblocks; ++b) {
		const uint64_t off = b * block_size;
		const uint32_t n = (uint32_t)(in_size - off < block_size ? in_size - off : block_size);
		XzbBlockResult res;
		const int r = hs_block_encode(in + off, n, opt, check, block_size, scratch.data(), cap, &res);
		if (r != XZB_OK) return r;
		if (pos + res.total_size > out_cap) return XZB_BUF_ERROR;
		memcpy(out + pos, scratch.data(), res.total_size);
		pos += res.total_size;
		unp[b] = res.unpadded_size; unc[b] = n;
	}
	const uint64_t isz = xzbi_index_encode(g_tab.crc32, unp.data(), unc.data(), nblocks, out + pos);
	pos += isz;
	pos += xzb_stream_footer(g_tab.crc32, out + pos, check, isz);
	*out_size = pos;
	return XZB_OK;
}

// LZMA2 payload decode with the product's decoder logic.
void hs_sha256(const uint8_t *in, uint32_t n, uint8_t out[32]) { xzb_sha256(in, n, out); }

int hs_lzma2_decode(const uint8_t *in, uint32_t in_size, uint32_t dict_size, uint8_t *out, uint32_t out_limit, uint32_t *in_used, uint32_t *out_used)
{
	XzbDec *d = (XzbDec *)malloc(sizeof(XzbDec));
	const int r = xzb_lzma2_decode(d, in, in_size, dict_size, out, out_limit, in_used, out_used, 0, 1);
	free(d);
	return r;
}

}  // extern "C"

// Delta / BCJ filters (xzb_filters.cuh) on the host: the same functions the kernels run, whole Block in place.
extern "C" void hostsim_filter_apply(uint32_t id, uint32_t arg, int enc, uint8_t *buf, uint32_t size)
{
	xzb_filter_apply_seq(XzbPreFilter{ id, arg }, buf, size, enc != 0);
}

// The container read side (xzb_frame.cuh), each entry point with its results flattened into integers.
extern "C" {

int hs_stream_header_decode(const uint8_t *in, uint32_t *check)
{
	tabs();
	return xzb_stream_header_decode(g_tab.crc32, in, check);
}

int hs_stream_footer_decode(const uint8_t *in, uint32_t *check, uint64_t *index_size)
{
	tabs();
	return xzb_stream_footer_decode(g_tab.crc32, in, check, index_size);
}

// out: hsize, flags, comp (value, end, status), uncomp (value, end, status)
int hs_block_framing(const uint8_t *h, uint64_t avail, uint64_t out[8])
{
	XzbBlockFraming f;
	if (!xzb_block_framing(h, avail, &f)) return 0;
	const uint64_t v[8] = { f.hsize, f.flags, f.comp.v, f.comp.end, (uint64_t)f.comp.st, f.uncomp.v, f.uncomp.end, (uint64_t)f.uncomp.st };
	memcpy(out, v, sizeof(v));
	return 1;
}

// out: hsize, comp, uncomp, dict_size, n_pre, then (id, arg) of each filter in front of LZMA2
int hs_block_header_decode(const uint8_t *h, uint64_t avail, uint64_t out[11])
{
	tabs();
	XzbBlockHeader hb;
	const int r = xzb_block_header_decode(g_tab.crc32, h, avail, &hb);
	if (r != XZB_OK) return r;
	out[0] = hb.hsize; out[1] = hb.comp; out[2] = hb.uncomp; out[3] = hb.dict_size; out[4] = hb.n_pre;
	for (uint32_t i = 0; i < hb.n_pre; ++i) { out[5 + 2 * i] = hb.pre[i].id; out[6 + 2 * i] = hb.pre[i].arg; }
	return r;
}

// want == NULL: nothing to compare against.  out: count, listed, end, stop
int hs_index_read(const uint8_t *in, uint64_t size, const xzb_index_record *want, uint64_t n_want, uint64_t out[4])
{
	tabs();
	const XzbIndexWant w{ want, n_want };
	XzbIndexRead x;
	const int r = xzb_index_read(g_tab.crc32, in, size, want != nullptr ? &w : nullptr, &x);
	out[0] = x.count; out[1] = x.listed; out[2] = x.end; out[3] = x.stop;
	return r;
}

}  // extern "C"
