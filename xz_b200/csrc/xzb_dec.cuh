// xzb_dec.cuh -- LZMA2 payload decoder for one .xz block (range decoder + dictionary copy).
//
// The output buffer of the block is the dictionary (whole block resident, never wraps), so
// dict_put / dict_repeat (lz/lz_decoder.h:202-300) are plain stores; `full` keeps the
// reference's meaning for distance validation (lz_decoder.h:147-151, lz_decoder.c:247-256).
// Reference: lzma/lzma2_decoder.c:55-230, lzma/lzma_decoder.c:234-1114,
// rangecoder/range_decoder.h:56-388.  Host/device; the CUDA kernel runs one .xz block per
// CUDA block (xzb_kernels.cu).
#pragma once
#include "xzb_common.cuh"

#ifdef __CUDA_ARCH__
#define XZB_SYNCWARP() __syncwarp()
#else
#define XZB_SYNCWARP() ((void)0)
#endif

// The decoder functions take (lane, nlanes): on the GPU all 32 lanes of a warp execute the same
// (uniform) bit decoding on a shared-memory model, lane 0 stores literals and the lanes share the
// match copies; on the host (tests/hostsim) lane = 0, nlanes = 1.
#define XZB_NEED_INPUT 100   // ran out of compressed bytes (truncated input)
#define XZB_NEED_OUTPUT 101  // decoder wants to write past the output limit

// Bit-tree arrays are 4-byte aligned: the decoder fetches both children of a node with one 32-bit load.
struct XzbLenDec {
	xzb_prob choice, choice2;
	alignas(4) xzb_prob low[XZB_POS_STATES_MAX][8];
	alignas(4) xzb_prob mid[XZB_POS_STATES_MAX][8];
	alignas(4) xzb_prob high[256];
};

struct XzbDec {  // lzma_lzma1_decoder, lzma/lzma_decoder.c:106-231
	alignas(4) xzb_prob literal[16 * 0x300];
	xzb_prob is_match[XZB_STATES][XZB_POS_STATES_MAX];
	xzb_prob is_rep[XZB_STATES], is_rep0[XZB_STATES], is_rep1[XZB_STATES], is_rep2[XZB_STATES];
	xzb_prob is_rep0_long[XZB_STATES][XZB_POS_STATES_MAX];
	alignas(4) xzb_prob dist_slot[XZB_DIST_STATES][XZB_DIST_SLOTS];
	xzb_prob pos_special[XZB_FULL_DISTANCES - XZB_DIST_MODEL_END];
	alignas(4) xzb_prob pos_align[XZB_ALIGN_SIZE];
	XzbLenDec match_len, rep_len;
	uint32_t state, rep0, rep1, rep2, rep3;
	uint32_t pos_mask, lc, literal_mask;
};

// Range decoder state (range_decoder.h:60-66) + input cursor: kept in registers by the caller.
// (A register window over the input with prefetched 8-byte words lost to the plain byte load below:
// the load hits L1 and the 64-bit shifts cost more than it.)
struct XzbRcd {
	uint32_t range, code;
	const uint8_t *in;
	uint32_t in_pos, in_end;
	uint32_t chunk_cut;    // the chunk's bytes are cut short by the end of the input
	uint32_t err;
};
XZB_HD uint32_t xzb_rcd_getbyte(XzbRcd *d) { return d->in[d->in_pos++]; }  // caller checked in_pos < in_end

XZB_HD_NOINLINE void xzb_dec_reset(XzbDec *d, uint32_t lc, uint32_t lp, uint32_t pb)  // lzma_decoder.c:1034-1114
{
	d->pos_mask = (1u << pb) - 1; d->lc = lc;
	d->literal_mask = (0x100u << lp) - (0x100u >> lc);
	const uint32_t coders = 0x300u << (lc + lp);
	for (uint32_t i = 0; i < coders; ++i) d->literal[i] = 1024;
	d->state = 0; d->rep0 = d->rep1 = d->rep2 = d->rep3 = 0;
	for (int i = 0; i < XZB_STATES; ++i) {
		for (uint32_t j = 0; j <= d->pos_mask; ++j) { d->is_match[i][j] = 1024; d->is_rep0_long[i][j] = 1024; }
		d->is_rep[i] = d->is_rep0[i] = d->is_rep1[i] = d->is_rep2[i] = 1024;
	}
	for (int i = 0; i < XZB_DIST_STATES; ++i) for (int j = 0; j < XZB_DIST_SLOTS; ++j) d->dist_slot[i][j] = 1024;
	for (int i = 0; i < XZB_FULL_DISTANCES - XZB_DIST_MODEL_END; ++i) d->pos_special[i] = 1024;
	for (int i = 0; i < XZB_ALIGN_SIZE; ++i) d->pos_align[i] = 1024;
	for (int k = 0; k < 2; ++k) {
		XzbLenDec *l = k ? &d->rep_len : &d->match_len;
		l->choice = l->choice2 = 1024;
		for (uint32_t ps = 0; ps < (1u << pb); ++ps) for (int i = 0; i < 8; ++i) { l->low[ps][i] = 1024; l->mid[ps][i] = 1024; }
		for (int i = 0; i < 256; ++i) l->high[i] = 1024;
	}
}

// rc_normalize, range_decoder.h:144-150.  Reading past the chunk's Compressed Size is
// corruption (lzma2_decoder.c:174-188); past the end of a truncated input is "need input".
XZB_HD void xzb_rcd_normalize(XzbRcd *d)
{
	if (d->range < (1u << 24)) {
		uint32_t b = 0;
		if (d->in_pos < d->in_end) b = xzb_rcd_getbyte(d);
		else if (!d->err) d->err = d->chunk_cut ? XZB_NEED_INPUT : XZB_DATA_ERROR;
		d->range <<= 8;
		d->code = (d->code << 8) | b;
	}
}

// rc_if_0 / rc_update_0 / rc_update_1, :152-214, with the probability already in a register
XZB_HD uint32_t xzb_rcd_bit_p(XzbRcd *d, xzb_prob *prob, uint32_t p)
{
	xzb_rcd_normalize(d);
	const uint32_t bound = (d->range >> 11) * p;
	if (d->code < bound) {
		d->range = bound;
		*prob = (xzb_prob)(p + ((2048 - p) >> 5));
		return 0;
	}
	d->range -= bound; d->code -= bound;
	*prob = (xzb_prob)(p - (p >> 5));
	return 1;
}
XZB_HD uint32_t xzb_rcd_bit(XzbRcd *d, xzb_prob *prob) { return xzb_rcd_bit_p(d, prob, *prob); }

XZB_HD uint32_t xzb_ld_pair(const xzb_prob *p)  // probabilities p[0] (low half) and p[1]; p is 4-byte aligned
{
#ifdef __CUDA_ARCH__
	return *reinterpret_cast<const uint32_t *>(p);
#else
	return (uint32_t)p[0] | ((uint32_t)p[1] << 16);
#endif
}

// rc_bittree / rc_bittree_rev index walk (node s has children 2s and 2s+1): both children are
// loaded while the bit of node s is still being decoded, which takes the shared-memory latency off
// the chain.  Returns the final node index (1 << bits) + bits-in-decoding-order.
XZB_HD uint32_t xzb_rcd_tree_walk(XzbRcd *d, xzb_prob *probs, const uint32_t bits)
{
	uint32_t s = 1, p = probs[1];
	for (uint32_t i = 0; i < bits; ++i) {
		uint32_t pair = 0;
		if (i + 1 < bits) pair = xzb_ld_pair(probs + 2 * s);
		const uint32_t bit = xzb_rcd_bit_p(d, &probs[s], p);
		s = (s << 1) | bit;
		p = bit ? pair >> 16 : pair & 0xFFFF;
	}
	return s;
}
XZB_HD uint32_t xzb_rcd_bittree(XzbRcd *d, xzb_prob *probs, uint32_t bits) { return xzb_rcd_tree_walk(d, probs, bits) - (1u << bits); }

XZB_HD uint32_t xzb_len_decode(XzbRcd *d, XzbLenDec *l, uint32_t pos_state)  // lzma_decoder.c:47-97
{
	if (xzb_rcd_bit(d, &l->choice) == 0) return 2 + xzb_rcd_bittree(d, l->low[pos_state], 3);
	if (xzb_rcd_bit(d, &l->choice2) == 0) return 2 + 8 + xzb_rcd_bittree(d, l->mid[pos_state], 3);
	return 2 + 16 + xzb_rcd_bittree(d, l->high, 8);
}

// One LZMA chunk (lzma_decode, lzma_decoder.c:234-1021; uncompressed size known, no EOPM).
XZB_HD_NOINLINE int xzb_lzma_chunk_decode(XzbDec *d, uint8_t *out, uint32_t *pos_ptr, uint32_t usize, uint32_t dict_start, uint32_t dict_size_r,
		uint32_t lane, uint32_t nlanes, XzbRcd *rcp)
{
	XzbRcd rc = *rcp;  // registers
	uint32_t pos = *pos_ptr;
	const uint32_t limit = pos + usize;
	rc.range = 0xFFFFFFFFu; rc.code = 0;  // rc_read_init, range_decoder.h:69-91
	for (int i = 0; i < 5; ++i) {
		if (rc.in_pos >= rc.in_end) { rcp->in_pos = rc.in_pos; return rc.chunk_cut ? XZB_NEED_INPUT : XZB_DATA_ERROR; }
		const uint32_t b = xzb_rcd_getbyte(&rc);
		if (i == 0 && b != 0x00) { rcp->in_pos = rc.in_pos; return XZB_DATA_ERROR; }
		rc.code = (rc.code << 8) | b;
	}
	rc.err = 0;
	uint32_t state = d->state, rep0 = d->rep0, rep1 = d->rep1, rep2 = d->rep2, rep3 = d->rep3;
	uint32_t prev = pos != dict_start ? out[pos - 1] : 0;  // previous byte, carried in a register (none right after a reset)
	while (pos < limit && !rc.err) {
		const uint32_t rel = pos - dict_start;  // dict.pos modulo 16 == bytes since dictionary reset modulo 16
		const uint32_t pos_state = rel & d->pos_mask;
		const uint32_t full = rel < dict_size_r ? rel : dict_size_r;
		// the byte a literal after a match is coded against: requested before the is_match bit is decoded
		uint32_t match_byte = 0;
		if (state >= XZB_LIT_STATES && full > rep0) match_byte = out[pos - rep0 - 1];
		if (xzb_rcd_bit(&rc, &d->is_match[state][pos_state]) == 0) {
			xzb_prob *probs = d->literal + 3u * ((((rel << 8) + prev) & d->literal_mask) << d->lc);
			uint32_t symbol = 1;
			if (state < XZB_LIT_STATES) {
				state = state <= 3 ? 0 : state - 3;
				symbol = xzb_rcd_tree_walk(&rc, probs, 8);
			} else {
				state = state <= 9 ? state - 3 : state - 6;
				uint32_t offset = 0x100;  // rc_matched_literal :270-300
				do {
					match_byte <<= 1;
					const uint32_t match_bit = match_byte & offset;
					const uint32_t bit = xzb_rcd_bit(&rc, &probs[offset + match_bit + symbol]);
					symbol = (symbol << 1) | bit;
					if (bit) offset &= match_bit; else offset &= ~match_bit;
				} while (symbol < 0x100);
			}
			if (lane == 0) out[pos] = (uint8_t)symbol;
			prev = symbol & 0xFF;
			++pos;
			XZB_SYNCWARP();
			continue;
		}
		uint32_t len;
		if (xzb_rcd_bit(&rc, &d->is_rep[state]) == 0) {
			state = state < XZB_LIT_STATES ? 7 : 10;
			rep3 = rep2; rep2 = rep1; rep1 = rep0;
			len = xzb_len_decode(&rc, &d->match_len, pos_state);
			const uint32_t slot = xzb_rcd_bittree(&rc, d->dist_slot[len < 6 ? len - 2 : 3], 6);
			if (slot < XZB_DIST_MODEL_START) {
				rep0 = slot;
			} else {
				uint32_t nbits = (slot >> 1) - 1;
				rep0 = 2 | (slot & 1);
				if (slot < XZB_DIST_MODEL_END) {
					rep0 <<= nbits;
					xzb_prob *probs = d->pos_special + rep0 - slot - 1;
					uint32_t sym = 1, off = 1;
					do {
						const uint32_t bit = xzb_rcd_bit(&rc, &probs[sym]);
						sym = (sym << 1) | bit;
						if (bit) rep0 += off;
						off <<= 1;
					} while (--nbits > 0);
				} else {
					nbits -= XZB_ALIGN_BITS;
					do {  // rc_direct, range_decoder.h:375-388
						xzb_rcd_normalize(&rc);
						rc.range >>= 1;
						rc.code -= rc.range;
						const uint32_t mask = 0u - (rc.code >> 31);
						rc.code += rc.range & mask;
						rep0 = (rep0 << 1) + (mask + 1);
					} while (--nbits > 0);
					rep0 <<= XZB_ALIGN_BITS;
					const uint32_t sym = xzb_rcd_tree_walk(&rc, d->pos_align, XZB_ALIGN_BITS);  // rc_bittree_rev: first bit decoded is bit 0
					rep0 += ((sym >> 3) & 1) | ((sym >> 1) & 2) | ((sym << 1) & 4) | ((sym << 3) & 8);
					if (rep0 == 0xFFFFFFFFu) { rc.err = XZB_DATA_ERROR; break; }  // EOPM is not allowed in LZMA2
				}
			}
			if (!(full > rep0)) { if (!rc.err) rc.err = XZB_DATA_ERROR; break; }
		} else {
			if (!(full > 0)) { if (!rc.err) rc.err = XZB_DATA_ERROR; break; }
			if (xzb_rcd_bit(&rc, &d->is_rep0[state]) == 0) {
				if (xzb_rcd_bit(&rc, &d->is_rep0_long[state][pos_state]) == 0) {
					state = state < XZB_LIT_STATES ? 9 : 11;
					if (!(full > rep0)) { if (!rc.err) rc.err = XZB_DATA_ERROR; break; }
					prev = out[pos - rep0 - 1];
					if (lane == 0) out[pos] = (uint8_t)prev;
					++pos;
					XZB_SYNCWARP();
					continue;
				}
			} else {
				uint32_t dist;
				if (xzb_rcd_bit(&rc, &d->is_rep1[state]) == 0) { dist = rep1; }
				else {
					if (xzb_rcd_bit(&rc, &d->is_rep2[state]) == 0) { dist = rep2; }
					else { dist = rep3; rep3 = rep2; }
					rep2 = rep1;
				}
				rep1 = rep0; rep0 = dist;
			}
			state = state < XZB_LIT_STATES ? 8 : 11;
			len = xzb_len_decode(&rc, &d->rep_len, pos_state);
			if (!(full > rep0)) { if (!rc.err) rc.err = XZB_DATA_ERROR; break; }
		}
		if (rc.err) break;
		// dict_repeat, lz_decoder.h:202-266; a match running past the chunk's size is corrupt
		if (len > limit - pos) { rc.err = XZB_DATA_ERROR; len = limit - pos; }
		// overlapping copies are periodic with period rep0 + 1, so every byte has a source that
		// was complete before this match started
		const uint32_t back = pos - rep0 - 1, period = rep0 + 1;
		for (uint32_t i = lane; i < len; i += nlanes) out[pos + i] = out[back + (i < period ? i : i % period)];
		pos += len;
		XZB_SYNCWARP();
		prev = out[pos - 1];
	}
	d->state = state; d->rep0 = rep0; d->rep1 = rep1; d->rep2 = rep2; d->rep3 = rep3;
	*pos_ptr = pos;
	if (!rc.err) xzb_rcd_normalize(&rc);  // lzma_decoder.c:661-690
	rcp->in_pos = rc.in_pos;
	if (rc.err) return (int)rc.err;
	if (rc.code != 0) return XZB_DATA_ERROR;
	return XZB_OK;
}

#ifdef __CUDACC__
__device__ int xzb_lzma_chunk_decode_w(XzbDec *d, uint8_t *out, uint32_t *pos_ptr, uint32_t usize, uint32_t dict_start, uint32_t dict_size_r,
		const uint32_t lane, XzbRcd *rcp);
#endif

// The dictionary size the LZ layer rounds to (lz_decoder.c:247-256).
XZB_HD uint32_t xzb_dict_size_r(uint32_t dict_size)
{
	const uint32_t r = dict_size < 4096 ? 4096 : dict_size;
	return r > 0xFFFFFFF0u ? 0xFFFFFFF0u : (r + 15) & ~15u;
}

// The chunk walk's state between two chunks (lzma2_decoder.c:23-52): what a resumed walk carries over.  dict_start is
// where the dictionary was last reset, in out[] positions; a resumed walk passes a virtual one (xzb_dec_resume.cuh).
struct XzbWalk {
	uint32_t need_properties, need_dictionary_reset;
	uint32_t lc, lp, pb;
	uint32_t dict_start;
	uint32_t dict_reset;   // set when a chunk reset the dictionary in this call
};
XZB_HD void xzb_walk_init(XzbWalk *w)
{
	w->need_properties = 1; w->need_dictionary_reset = 1;
	w->lc = w->lp = w->pb = 0; w->dict_start = 0; w->dict_reset = 0;
}

// lzma2_decode, lzma/lzma2_decoder.c:55-230, over whole or cut chunks from in[0 .. in_size), writing out[pos0 ..
// out_limit).  Returns XZB_OK at the end marker, XZB_DATA_ERROR, XZB_NEED_INPUT or XZB_NEED_OUTPUT; the walk state
// *w is read on entry and written back on return.  (Inlined into its two callers below, so that the whole-Block decode
// keeps the walk state in registers as a plain local.)
XZB_HD int xzb_lzma2_walk_body(XzbDec *d, XzbWalk *w, const uint8_t *in, uint32_t in_size, uint32_t dict_size_r,
		uint8_t *out, uint32_t pos0, uint32_t out_limit, uint32_t *in_used, uint32_t *out_used, uint32_t lane, uint32_t nlanes)
{
	uint32_t in_pos = 0, pos = pos0, dict_start = w->dict_start;
	bool need_properties = w->need_properties != 0, need_dictionary_reset = w->need_dictionary_reset != 0;
	uint32_t lc = w->lc, lp = w->lp, pb = w->pb;
	int ret;
	for (;;) {
		if (in_pos >= in_size) { ret = XZB_NEED_INPUT; break; }
		const uint32_t control = in[in_pos++];
		if (control == 0x00) { ret = XZB_OK; break; }
		if (control >= 0xE0 || control == 1) { need_properties = true; need_dictionary_reset = true; }
		else if (need_dictionary_reset) { ret = XZB_DATA_ERROR; break; }
		const bool is_lzma = control >= 0x80;
		bool new_props = false, state_reset = false;
		if (is_lzma) {
			if (control >= 0xC0) { need_properties = false; new_props = true; }
			else if (need_properties) { ret = XZB_DATA_ERROR; break; }
			else if (control >= 0xA0) state_reset = true;
		} else if (control > 2) { ret = XZB_DATA_ERROR; break; }
		if (need_dictionary_reset) { need_dictionary_reset = false; dict_start = pos; w->dict_reset = 1; }
		uint32_t usize = 0;
		if (is_lzma) {
			if (in_size - in_pos < 2) { in_pos = in_size; ret = XZB_NEED_INPUT; break; }
			usize = ((control & 0x1F) << 16) + ((uint32_t)in[in_pos] << 8) + in[in_pos + 1] + 1;
			in_pos += 2;
		}
		if (in_size - in_pos < 2) { in_pos = in_size; ret = XZB_NEED_INPUT; break; }
		const uint32_t csize = ((uint32_t)in[in_pos] << 8) + in[in_pos + 1] + 1;
		in_pos += 2;
		if (!is_lzma) {  // SEQ_COPY: dict_write, lz_decoder.h:283-297
			uint32_t n = csize;
			bool short_in = false, short_out = false;
			if (n > in_size - in_pos) { n = in_size - in_pos; short_in = true; }
			if (n > out_limit - pos) { n = out_limit - pos; short_out = true; short_in = false; }
			for (uint32_t i = lane; i < n; i += nlanes) out[pos + i] = in[in_pos + i];
			pos += n; in_pos += n;
			XZB_SYNCWARP();
			if (short_out) { ret = XZB_NEED_OUTPUT; break; }
			if (short_in) { ret = XZB_NEED_INPUT; break; }
			continue;
		}
		if (new_props) {
			if (in_pos >= in_size) { ret = XZB_NEED_INPUT; break; }
			uint32_t byte = in[in_pos++];  // lzma_lzma_lclppb_decode, lzma_decoder.c:1198-1211
			if (byte > (4 * 5 + 4) * 9 + 8) { ret = XZB_DATA_ERROR; break; }
			pb = byte / (9 * 5); byte -= pb * 9 * 5; lp = byte / 9; lc = byte - lp * 9;
			if (lc + lp > 4) { ret = XZB_DATA_ERROR; break; }
			xzb_dec_reset(d, lc, lp, pb);
		} else if (state_reset) {
			xzb_dec_reset(d, lc, lp, pb);
		}
		XzbRcd rc;  // SEQ_LZMA :165-196
		rc.in = in; rc.in_pos = in_pos; rc.range = 0; rc.code = 0; rc.err = 0;
		const uint32_t chunk_start = in_pos;
		rc.chunk_cut = csize > in_size - in_pos;
		rc.in_end = rc.chunk_cut ? in_size : in_pos + csize;
		uint32_t want = usize; bool short_out = false;
		if (want > out_limit - pos) { want = out_limit - pos; short_out = true; }
#if defined(__CUDA_ARCH__) && !defined(XZB_DEC_GENERIC)
		ret = xzb_lzma_chunk_decode_w(d, out, &pos, want, dict_start, dict_size_r, lane, &rc);   // xzb_dec_warp.cuh
#else
		ret = xzb_lzma_chunk_decode(d, out, &pos, want, dict_start, dict_size_r, lane, nlanes, &rc);
#endif
		in_pos = rc.in_pos;
		if (short_out && (ret == XZB_OK || ret == XZB_DATA_ERROR)) { ret = XZB_NEED_OUTPUT; break; }
		if (ret != XZB_OK) break;
		if (in_pos - chunk_start != csize) { ret = XZB_DATA_ERROR; break; }  // :190-193
	}
	w->need_properties = need_properties; w->need_dictionary_reset = need_dictionary_reset;
	w->lc = lc; w->lp = lp; w->pb = pb; w->dict_start = dict_start;
	*in_used = in_pos; *out_used = pos - pos0;
	return ret;
}

// A run of chunks of a Block decoded piece by piece (xzb_dec_resume.cuh).
XZB_HD_NOINLINE int xzb_lzma2_walk(XzbDec *d, XzbWalk *w, const uint8_t *in, uint32_t in_size, uint32_t dict_size_r,
		uint8_t *out, uint32_t pos0, uint32_t out_limit, uint32_t *in_used, uint32_t *out_used, uint32_t lane, uint32_t nlanes)
{
	return xzb_lzma2_walk_body(d, w, in, in_size, dict_size_r, out, pos0, out_limit, in_used, out_used, lane, nlanes);
}

// One whole Block's LZMA2 data into out[0 .. out_limit).
XZB_HD_NOINLINE int xzb_lzma2_decode(XzbDec *d, const uint8_t *in, uint32_t in_size, uint32_t dict_size,
		uint8_t *out, uint32_t out_limit, uint32_t *in_used, uint32_t *out_used, uint32_t lane, uint32_t nlanes)
{
	XzbWalk w;
	xzb_walk_init(&w);
	return xzb_lzma2_walk_body(d, &w, in, in_size, xzb_dict_size_r(dict_size), out, 0, out_limit, in_used, out_used, lane, nlanes);
}
