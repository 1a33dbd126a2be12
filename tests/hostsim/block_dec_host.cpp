// tests/hostsim/block_dec_host.cpp -- TEST HARNESS (tests only): the resumable Block decoder of xz_b200/csrc/xzb_dec_resume.cuh
// (XzbBlockDec, the body of xzb_block_decoder_*) over a host backend, compiled with g++ so that
// tests/test_block_decoder_cpu.py can drive it without a GPU: the same window, piece, hand-out and verdict logic, with the
// host form of the chunk decoder, CRC and SHA-256 in place of the kernels.  Not part of the product and never used as a
// fallback.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../xz_b200/csrc/xzb_common.cuh"
#include "../../xz_b200/csrc/xzb_frame.cuh"
#include "../../xz_b200/csrc/xzb_params.h"
#include "../../xz_b200/csrc/xzb_dec_resume.cuh"

static const XzbHostTables &tables()
{
	static XzbHostTables t;
	static bool init = false;
	if (!init) { xzb_make_tables(&t); init = true; }
	return t;
}

struct HostBackend {
	std::vector<uint8_t> win;
	XzbDec *d = nullptr;
	XzbSha256State sha;
	uint64_t moved = 0;
	HostBackend() { d = (XzbDec *)calloc(1, sizeof(XzbDec)); xzb_sha256_init(&sha); }
	~HostBackend() { free(d); }
	int reserve(uint64_t cap, uint32_t keep) { (void)keep; win.resize(cap); return XZB_OK; }
	int move(uint32_t dst, uint32_t src, uint32_t n)
	{
		memmove(win.data() + dst, win.data() + src, n);
		memset(win.data() + dst + n, 0xA5, src - dst);   // the bytes the history left behind
		stale = 0; moved += n;
		return XZB_OK;
	}
	uint32_t stale = 0;   // window bytes [0, stale) are garbled already
	int decode(const uint8_t *in, uint32_t in_size, uint32_t pos, uint32_t out_limit, XzbResume *r, uint32_t *iu, uint32_t *ou, int *ret)
	{
		// what the decoder may no longer need is garbled first, so that a read of it shows in the output: window bytes
		// older than min(bytes out, dict_size_r), and the model when the piece's first chunk resets it (the kernel
		// xzb_k_decode_resume does not load it then)
		const uint64_t hist = r->out_total < r->dict_size_r ? r->out_total : r->dict_size_r;
		if (pos - hist > stale) { memset(win.data() + stale, 0xA5, pos - hist - stale); stale = (uint32_t)(pos - hist); }
		if (in_size != 0 && (in[0] >= 0xA0 || r->walk.need_properties)) memset(d, 0x5A, sizeof(XzbDec));
		*ret = xzb_resume_piece(d, r, in, in_size, win.data(), pos, out_limit, iu, ou, 0, 1);
		return XZB_OK;
	}
	int check(uint32_t id, uint32_t pos, uint32_t n, uint64_t *crc)
	{
		const uint8_t *p = win.data() + pos;
		if (id == 10) { xzb_sha256_update(&sha, p, n); return XZB_OK; }
		uint64_t c;
		if (id == 1) { const uint32_t *t = tables().crc32; c = 0xFFFFFFFFull; for (uint32_t i = 0; i < n; ++i) c = t[(c ^ p[i]) & 0xFF] ^ (c >> 8); c ^= 0xFFFFFFFFull; }
		else { const uint64_t *t = tables().crc64; c = ~0ull; for (uint32_t i = 0; i < n; ++i) c = t[(c ^ p[i]) & 0xFF] ^ (c >> 8); c ^= ~0ull; }
		*crc = c;
		return XZB_OK;
	}
	int sha_final(uint8_t out[32]) { xzb_sha256_final(&sha, out); return XZB_OK; }
	int fetch(uint8_t *dst, uint32_t pos, uint64_t n) { memcpy(dst, win.data() + pos, n); return XZB_OK; }
};

extern "C" {

// Decodes the Block blk[0 .. blk_size) (Block Header .. Check field) with the resumable decoder, as a caller that streams
// it would: the input it has grows to cuts[0], cuts[1], .. and finally blk_size (LZMA_FINISH from then on), and it takes
// the output out_step bytes per call (0: its whole buffer).  piece_in / piece_out: the decoder's piece caps (0: default).
// stats: pieces, slides, bytes slid, largest history slid, dict_size_r, calls, largest window.  Returns the final code
// (1 = end of Block) with *out_size bytes of output and *in_used bytes consumed.
int bd_run(const uint8_t *blk, uint64_t blk_size, uint32_t check, uint32_t flags, const uint64_t *cuts, uint32_t ncuts, uint64_t out_step,
		uint64_t piece_in, uint64_t piece_out, uint8_t *out, uint64_t out_cap, uint64_t *out_size, uint64_t *in_used, uint64_t *stats,
		xzb_index_record *rec)
{
	*out_size = 0; *in_used = 0;
	XzbBlockHeader hb;
	int r = xzb_block_header_decode(tables().crc32, blk, blk_size, &hb);
	if (r != XZB_OK) return r;
	if (hb.n_pre != 0) return XZB_OPTIONS_ERROR;
	XzbBlockDec<HostBackend> *bd = new XzbBlockDec<HostBackend>();
	bd->init(tables().crc32, tables().crc64, hb, check, flags);
	if (piece_in) bd->piece_in = piece_in;
	if (piece_out) bd->piece_out = piece_out;
	uint64_t consumed = hb.hsize, calls = 0;
	uint32_t k = 0;
	uint64_t have = ncuts ? std::min<uint64_t>(std::max<uint64_t>(cuts[0], consumed), blk_size) : blk_size;
	for (;;) {
		const uint64_t cap = out_step ? std::min(out_step, out_cap - *out_size) : out_cap - *out_size;
		uint64_t iu = 0, os = 0;
		r = bd->code(blk + consumed, have - consumed, &iu, out + *out_size, cap, &os, have == blk_size);
		++calls;
		consumed += iu; *out_size += os;
		if (r != XZB_OK) break;
		if (iu == 0 && os == 0) {
			if (have == blk_size) { r = XZB_PROG_ERROR; break; }   // no progress with all input in: a decoder bug
			while (k < ncuts && cuts[k] <= have) ++k;
			have = k < ncuts ? std::min(cuts[k], blk_size) : blk_size;
		}
		if (calls > 100000000ull) { r = XZB_PROG_ERROR; break; }
	}
	*in_used = consumed;
	bd->record(rec);
	stats[0] = bd->pieces; stats[1] = bd->slides; stats[2] = bd->bytes_slid; stats[3] = bd->max_history;
	stats[4] = bd->r.dict_size_r; stats[5] = calls; stats[6] = bd->max_window;
	delete bd;
	return r;
}

}  // extern "C"
