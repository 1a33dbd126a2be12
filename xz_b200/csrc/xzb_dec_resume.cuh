// xzb_dec_resume.cuh -- one LZMA2 Block decoded piece by piece (a run of whole chunks at a time) in bounded memory, for
// unsized Blocks and Blocks too large for a whole-Block job.  Reference: common/block_decoder.c:64-200 (the Block),
// lzma/lzma2_decoder.c:55-230 (the chunk walk), lz/lz_decoder.c:128-160 (the dictionary that outlives a call).
//
// Every LZMA2 chunk starts a fresh range decoder, and xzb_lzma2_walk ends a chunk with its copies flushed, so between two
// chunks the decoder's whole state is: the probability model with state and rep0..3 (XzbDec), the walk flags (XzbWalk),
// the bytes since the last dictionary reset, and the last min(dict_size_r, bytes out) bytes of output.  A piece is
// decoded by the same xzb_lzma2_walk as a whole Block; it writes into a window that holds that history and room for the
// piece, and gets a virtual dict_start (xzb_resume_piece) so that the chunk decoder's 32-bit positions give the same
// pos_state, literal position and distance limit as a decode of the whole Block would, past 4 GiB included.
//
//   XzbResume        the per-job record between pieces (with the model it lives in HBM for xzb_k_decode_resume)
//   xzb_chunk_run    how many bytes of whole chunks are at the front of the input, and the output they can produce
//   xzb_resume_piece one piece on one warp (device) or one thread (host, tests/hostsim)
//   XzbBlockDec<B>   the Block decoder behind xzb_block_decoder_*: window, pieces, output hand-out, Block Padding,
//                    Check field and verdicts; B supplies the memory and the decode / check steps (GPU or host).
#pragma once
#include "xzb_common.cuh"
#include "xzb_dec.cuh"
#include "xzb_frame.cuh"
#include "xzb_sha256.cuh"
#include <cstring>

struct XzbResume {
	XzbWalk walk;
	uint32_t dict_size_r;
	uint64_t out_total;   // bytes out so far
	uint64_t rel;         // bytes out since the last dictionary reset
	uint64_t in_total;    // compressed bytes in so far
};

XZB_HD void xzb_resume_init(XzbResume *r, uint32_t dict_size)
{
	xzb_walk_init(&r->walk);
	r->dict_size_r = xzb_dict_size_r(dict_size);
	r->out_total = r->rel = r->in_total = 0;
}

// The distance from the virtual dict_start to the next output byte: == rel modulo 16 and min(v, dict_size_r) ==
// min(rel, dict_size_r).  These are the only two things the chunk decoder reads of rel.
XZB_HD uint64_t xzb_resume_vrel(const XzbResume *r)
{
	return r->rel < r->dict_size_r ? r->rel : (uint64_t)r->dict_size_r + (r->rel & 15);
}

// Decodes in[0 .. in_size) into win[pos .. out_limit); win[pos - min(out_total, dict_size_r) .. pos) holds the history.
// *r is updated for the bytes consumed and produced.  Same return values as xzb_lzma2_walk.
XZB_HD int xzb_resume_piece(XzbDec *d, XzbResume *r, const uint8_t *in, uint32_t in_size, uint8_t *win, uint32_t pos,
		uint32_t out_limit, uint32_t *in_used, uint32_t *out_used, uint32_t lane, uint32_t nlanes)
{
	XzbWalk w = r->walk;
	w.dict_start = pos - (uint32_t)xzb_resume_vrel(r);   // may wrap below 0: only differences of positions are used
	w.dict_reset = 0;
	const int ret = xzb_lzma2_walk(d, &w, in, in_size, r->dict_size_r, win, pos, out_limit, in_used, out_used, lane, nlanes);
	r->rel = w.dict_reset ? (uint64_t)(pos + *out_used - w.dict_start) : r->rel + *out_used;
	r->walk = w;
	r->out_total += *out_used;
	r->in_total += *in_used;
	return ret;
}

// Whole chunks at the front of in[0 .. avail) (lzma2_decoder.c:55-160 header layout).  Stops before a chunk that is not
// all there, after the end marker, after a control byte no chunk has (the walk reports it), or before the chunk that
// would take the run past max_in bytes or max_out bytes of output (a run has at least one chunk).
struct XzbChunkRun {
	uint64_t bytes;       // whole chunks (and the end marker / a bad control byte)
	uint64_t out_bound;   // the output they can produce: the sum of the headers' unpacked sizes
	uint32_t chunks;
	uint32_t end;         // the end marker is included
};
XZB_HD void xzb_chunk_run(const uint8_t *in, uint64_t avail, uint64_t max_in, uint64_t max_out, XzbChunkRun *r)
{
	uint64_t p = 0, out = 0;
	r->chunks = 0; r->end = 0;
	while (p < avail) {
		const uint32_t c = in[p];
		if (c == 0x00) { p += 1; r->end = 1; break; }
		uint64_t hdr, usize, csize;
		if (c >= 0x80) {
			hdr = c >= 0xC0 ? 6 : 5;
			if (avail - p < 5) break;
			usize = ((uint64_t)(c & 0x1F) << 16) + ((uint32_t)in[p + 1] << 8) + in[p + 2] + 1;
			csize = ((uint32_t)in[p + 3] << 8) + in[p + 4] + 1;
		} else if (c <= 2) {
			hdr = 3;
			if (avail - p < 3) break;
			csize = ((uint32_t)in[p + 1] << 8) + in[p + 2] + 1;
			usize = csize;
		} else {
			p += 1; ++r->chunks;
			break;
		}
		if (avail - p < hdr + csize) break;
		if (r->chunks != 0 && (p + hdr + csize > max_in || out + usize > max_out)) break;
		p += hdr + csize; out += usize; ++r->chunks;
	}
	r->bytes = p; r->out_bound = out;
}

// (host code from here on)
// CRC32 / CRC64 of a message that arrives in pieces, on the host from the pieces' CRCs: crc(A || B) =
// Z^|B| (crc(A)) ^ crc(B), where Z advances the register over one zero byte (the operator xzb_k_crc builds per slice),
// here raised to |B| by repeated squaring as a 64 x 64 matrix over GF(2).
struct XzbCrcCombine {
	uint64_t z[64];   // one zero byte
	template <class T> void init(const T *table)
	{
		for (int j = 0; j < 64; ++j) { const uint64_t x = 1ull << j; z[j] = (uint64_t)table[x & 0xFF] ^ (x >> 8); }
	}
	static uint64_t apply(const uint64_t *m, uint64_t v)
	{
		uint64_t r = 0;
		for (int j = 0; v; ++j, v >>= 1) if (v & 1) r ^= m[j];
		return r;
	}
	uint64_t advance(uint64_t crc, uint64_t len) const
	{
		uint64_t m[64], t[64];
		memcpy(m, z, sizeof(m));
		while (len) {
			if (len & 1) crc = apply(m, crc);
			len >>= 1;
			if (len) { for (int j = 0; j < 64; ++j) t[j] = apply(m, m[j]); memcpy(m, t, sizeof(m)); }
		}
		return crc;
	}
	uint64_t combine(uint64_t crc_a, uint64_t crc_b, uint64_t len_b) const { return advance(crc_a, len_b) ^ crc_b; }
};

// The Block decoder.  B provides (all positions are window offsets, all sizes in bytes):
//   int reserve(uint64_t cap, uint32_t keep)   window of at least cap bytes, its first `keep` bytes preserved
//   int move(uint32_t dst, uint32_t src, uint32_t n)   dst < src; the ranges overlap only when the window cannot grow
//   int decode(const uint8_t *in, uint32_t in_size, uint32_t pos, uint32_t out_limit, XzbResume *r,
//              uint32_t *in_used, uint32_t *out_used, int *ret)   one piece (xzb_resume_piece)
//   int check(uint32_t id, uint32_t pos, uint32_t n, uint64_t *crc)   CRC32 / CRC64 (id 1 / 4) of window bytes, or feed
//              them to the running SHA-256 (id 10)
//   int sha_final(uint8_t out[32])
//   int fetch(uint8_t *dst, uint32_t pos, uint64_t n)   window bytes to the caller
// Each returns XZB_OK or an error of the device / memory, which ends the Block with that code.
template <class B> struct XzbBlockDec {
	B be;
	XzbBlockHeader hb;
	uint32_t check = 0, csize = 0, verify = 1;
	uint64_t piece_in = 1u << 20;      // compressed bytes per piece (at least one chunk)
	uint64_t piece_out = 64u << 20;    // output bound per piece (at least one chunk)
	XzbResume r;
	uint64_t win_cap = 0;
	uint32_t win_pos = 0;      // end of the decoded bytes in the window
	uint32_t deliv = 0;        // the first byte not handed out yet
	int ret = XZB_OK;          // latched verdict
	uint32_t phase = 0;        // 0 LZMA2 data, 1 Block Padding + Check, 2 done
	uint32_t tail_have = 0;    // bytes of Block Padding + Check field consumed
	uint8_t stored[64];        // the Check field as read
	uint64_t crc = 0;
	XzbCrcCombine comb;
	// counters for tests and the probe
	uint64_t pieces = 0, slides = 0, bytes_slid = 0, max_history = 0, max_window = 0;

	static const uint32_t WIN_LIMIT = 0xFFFFFFF0u;   // window positions are 32-bit (the chunk decoder's)

	int init(const uint32_t *crc32_table, const uint64_t *crc64_table, const XzbBlockHeader &h, uint32_t check_id, uint32_t flags)
	{
		hb = h; check = check_id;
		csize = xzb_check_field_size(check);
		verify = !(flags & XZB_DEC_IGNORE_CHECK) && (check == 1 || check == 4 || check == 10);
		if (check == 1) comb.init(crc32_table);
		if (check == 4) comb.init(crc64_table);
		xzb_resume_init(&r, hb.dict_size);
		return XZB_OK;
	}

	// Room for `bound` more bytes behind the history.  The history moves to the front only once at least as many bytes
	// as it holds were written behind it since the window's start -- so a move of at most a dictionary is paid for by at
	// least as much output, and source and destination do not overlap -- or when the window cannot grow any more.
	// Otherwise the window grows (doubling) towards twice the dictionary plus a piece, where the first rule always holds.
	int make_room(uint64_t bound)
	{
		const uint64_t hist = r.out_total < r.dict_size_r ? r.out_total : r.dict_size_r;
		if (xzb_resume_vrel(&r) + bound > 0xFFFFFFFFull || hist + bound > WIN_LIMIT) return XZB_MEM_ERROR;
		if (win_pos + bound <= win_cap) return XZB_OK;
		uint64_t target = 2 * (uint64_t)r.dict_size_r + (bound > piece_out ? bound : piece_out);
		if (target > WIN_LIMIT) target = WIN_LIMIT;
		if (win_pos > hist && (win_pos - hist >= hist || win_pos + bound > target)) {
			const int e = be.move(0, (uint32_t)(win_pos - hist), (uint32_t)hist);
			if (e != XZB_OK) return e;
			++slides; bytes_slid += hist;
			if (hist > max_history) max_history = hist;
			win_pos = deliv = (uint32_t)hist;
		}
		if (win_pos + bound > win_cap) {
			uint64_t want = 2 * win_cap < target ? 2 * win_cap : target;
			if (want < win_pos + bound) want = win_pos + bound;
			const int e = be.reserve(want, win_pos);
			if (e != XZB_OK) return e;
			win_cap = want;
			if (want > max_window) max_window = want;
		}
		return XZB_OK;
	}

	int fail(int code) { ret = code; return code; }

	// One piece of LZMA2 data from in[0 .. avail); returns false when it needs more input first.
	bool step_data(const uint8_t *in, uint64_t avail, uint64_t *used, bool finish)
	{
		const uint64_t lim = hb.comp != UINT64_MAX ? hb.comp - r.in_total : UINT64_MAX;
		XzbChunkRun run;
		xzb_chunk_run(in, avail < lim ? avail : lim, piece_in, piece_out, &run);
		uint64_t piece = run.bytes, bound = run.out_bound;
		bool cut = false, truncated = true;
		if (run.chunks == 0 && !run.end) {
			// no whole chunk: the Compressed Size ends inside it (corrupt), or the input does (truncated) at LZMA_FINISH
			if (lim <= avail) { piece = lim; cut = true; truncated = false; }
			else if (finish) { piece = avail; cut = true; }
			else return false;
			bound = 1u << 21;   // a chunk's largest unpacked size
		}
		if (piece > 0xFFFFFFFFull) piece = 0xFFFFFFFFull;   // (only a Compressed Size limit can make it that large)
		if (hb.uncomp != UINT64_MAX && bound > hb.uncomp - r.out_total) bound = hb.uncomp - r.out_total;
		int e = make_room(bound);
		if (e != XZB_OK) { fail(e); return true; }
		uint32_t iu = 0, ou = 0;
		int dr = XZB_OK;
		e = be.decode(in, (uint32_t)piece, win_pos, (uint32_t)(win_pos + bound), &r, &iu, &ou, &dr);
		if (e != XZB_OK) { fail(e); return true; }
		++pieces;
		if (verify && ou != 0) {
			uint64_t c = 0;
			e = be.check(check, win_pos, ou, &c);
			if (e != XZB_OK) { fail(e); return true; }
			if (check != 10) crc = comb.combine(crc, c, ou);
		}
		win_pos += ou;
		*used += iu;
		if (dr == XZB_OK) {
			phase = 1;
			if ((hb.comp != UINT64_MAX && r.in_total != hb.comp) || (hb.uncomp != UINT64_MAX && r.out_total != hb.uncomp)) fail(XZB_DATA_ERROR);
		} else if (dr == XZB_NEED_INPUT) {
			if (cut) fail(truncated ? XZB_BUF_ERROR : XZB_DATA_ERROR);
		} else if (dr == XZB_NEED_OUTPUT) {
			fail(XZB_DATA_ERROR);   // only the Uncompressed Size limits a piece's output
		} else {
			fail(dr);
		}
		return true;
	}

	// Block Padding and the Check field (block_decoder.c:146-196); returns false when it needs more input first.
	bool step_tail(const uint8_t *in, uint64_t avail, uint64_t *used, bool finish)
	{
		const uint64_t npad = (4 - (r.in_total & 3)) & 3;
		while (tail_have < npad + csize) {
			if (*used >= avail) {
				if (!finish) return false;
				fail(XZB_BUF_ERROR);
				return true;
			}
			const uint8_t b = in[(*used)++];
			if (tail_have < npad) { if (b != 0x00) { fail(XZB_DATA_ERROR); return true; } }
			else stored[tail_have - npad] = b;
			++tail_have;
		}
		if (verify) {
			uint8_t want[32];
			if (check == 10) {
				const int e = be.sha_final(want);
				if (e != XZB_OK) { fail(e); return true; }
			} else {
				for (uint32_t i = 0; i < csize; ++i) want[i] = (uint8_t)(crc >> (8 * i));
			}
			for (uint32_t i = 0; i < csize; ++i) if (want[i] != stored[i]) { fail(XZB_DATA_ERROR); return true; }
		}
		phase = 2;
		return true;
	}

	// xzb_block_decoder_code
	int code(const uint8_t *in, uint64_t in_size, uint64_t *in_used, uint8_t *out, uint64_t out_cap, uint64_t *out_size, bool finish)
	{
		*in_used = 0; *out_size = 0;
		for (;;) {
			const uint64_t n = (uint64_t)(win_pos - deliv) < out_cap - *out_size ? (uint64_t)(win_pos - deliv) : out_cap - *out_size;
			if (n) {
				const int e = be.fetch(out + *out_size, deliv, n);
				if (e != XZB_OK) return fail(e);
				deliv += (uint32_t)n; *out_size += n;
			}
			if (deliv != win_pos) return XZB_OK;   // the caller's buffer is full
			if (ret != XZB_OK) return ret;
			if (phase == 2) return 1;              // LZMA_STREAM_END
			const bool more = phase == 0 ? step_data(in + *in_used, in_size - *in_used, in_used, finish)
			                             : step_tail(in, in_size, in_used, finish);
			if (!more) return XZB_OK;
		}
	}

	void record(xzb_index_record *rec) const
	{
		rec->unpadded_size = hb.hsize + r.in_total + csize;
		rec->uncompressed_size = r.out_total;
	}
};
