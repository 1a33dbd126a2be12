// xzb_dec_warp.cuh -- the LZMA chunk decoder of xzb_dec.cuh restated for one GPU warp (device only).
//
// Same bit-for-bit decisions and the same verdicts as xzb_lzma_chunk_decode (lzma_decode, lzma/lzma_decoder.c:234-1021);
// what changes is what sits on the serial chain of the range decoder (range_decoder.h:144-214):
//   * the next compressed byte is always preloaded in a register, so a normalisation (one bit in eight or so, behind
//     one compare-and-branch on the common path) is two shifts and an OR, and the load of the byte after it has
//     several bits' time to complete (ncu, profiles/r02_decode_ncu.txt: a fully predicated normalisation executed on
//     every bit cost 55 % of the kernel's issue slots and was dropped);
//   * dict_repeat (lz_decoder.h:202-266) is split: the lanes LOAD the source bytes of a match (<= 32 bytes: one per
//     lane) when it is decoded and keep them in registers; they are STORED when the next match is decoded (its source
//     may lie in this one's destination), when a literal needs them, or at the end of the chunk.  The window read
//     (L2 latency for far distances) so overlaps the decoding of the following symbol instead of stalling it;
//   * the byte before a literal and the byte it is matched against come out of those registers (one shuffle) when
//     they belong to the pending copy, and are only looked at when the symbol really is a literal.
#pragma once
#include "xzb_dec.cuh"

struct XzbRcw {   // range decoder (range_decoder.h:60-66) + input cursor + the preloaded byte
	uint32_t range, code, nb;
	const uint8_t *cur, *end;   // nb == (cur < end ? *cur : 0): the next byte, not consumed yet
	uint32_t err;               // sticky: ran past the chunk's bytes
};

__device__ __forceinline__ void xzb_rcw_normalize(XzbRcw &r)
{
	if (r.range < (1u << 24)) {
		r.range <<= 8;
		r.code = (r.code << 8) | r.nb;
		if (r.cur < r.end) { ++r.cur; r.nb = r.cur < r.end ? (uint32_t)*r.cur : 0u; }
		else r.err = 1;
	}
}
__device__ __forceinline__ uint32_t xzb_rcw_bit_p(XzbRcw &r, xzb_prob *prob, const uint32_t p)
{
	xzb_rcw_normalize(r);
	const uint32_t bound = (r.range >> 11) * p;
	const bool bit = r.code >= bound;
	r.range = bit ? r.range - bound : bound;
	r.code = bit ? r.code - bound : r.code;
	*prob = (xzb_prob)(bit ? p - (p >> 5) : p + ((2048 - p) >> 5));
	return bit ? 1u : 0u;
}
__device__ __forceinline__ uint32_t xzb_rcw_bit(XzbRcw &r, xzb_prob *prob) { return xzb_rcw_bit_p(r, prob, *prob); }
// rc_bittree / rc_bittree_rev walk with both children of the next node fetched while this node's bit is decoded
__device__ __forceinline__ uint32_t xzb_rcw_tree_walk(XzbRcw &r, xzb_prob *probs, const uint32_t bits)
{
	uint32_t s = 1, p = probs[1];
	// unrolled: the decode chain is one warp's instruction stream, and the rolled loop adds its loop overhead to every bit
#pragma unroll
	for (uint32_t i = 0; i < bits; ++i) {
		uint32_t pair = 0;
		if (i + 1 < bits) pair = *reinterpret_cast<const uint32_t *>(probs + 2 * s);
		const uint32_t bit = xzb_rcw_bit_p(r, &probs[s], p);
		s = (s << 1) | bit;
		p = bit ? pair >> 16 : pair & 0xFFFF;
	}
	return s;
}
__device__ __forceinline__ uint32_t xzb_rcw_len(XzbRcw &r, XzbLenDec *l, uint32_t pos_state)  // lzma_decoder.c:47-97
{
	if (xzb_rcw_bit(r, &l->choice) == 0) return 2 + xzb_rcw_tree_walk(r, l->low[pos_state], 3) - 8;
	if (xzb_rcw_bit(r, &l->choice2) == 0) return 2 + 8 + xzb_rcw_tree_walk(r, l->mid[pos_state], 3) - 8;
	return 2 + 16 + xzb_rcw_tree_walk(r, l->high, 8) - 256;
}

// One LZMA chunk on one warp; arguments and return values as xzb_lzma_chunk_decode.
__device__ __noinline__ int xzb_lzma_chunk_decode_w(XzbDec *d, uint8_t *out, uint32_t *pos_ptr, uint32_t usize, uint32_t dict_start, uint32_t dict_size_r,
		const uint32_t lane, XzbRcd *rcp)
{
	XzbRcw rc;
	rc.cur = rcp->in + rcp->in_pos; rc.end = rcp->in + rcp->in_end; rc.err = 0;
	const uint32_t chunk_cut = rcp->chunk_cut;
	uint32_t pos = *pos_ptr;
	const uint32_t limit = pos + usize;
	rc.range = 0xFFFFFFFFu; rc.code = 0;  // rc_read_init, range_decoder.h:69-91
	for (int i = 0; i < 5; ++i) {
		if (rc.cur >= rc.end) { rcp->in_pos = (uint32_t)(rc.cur - rcp->in); return chunk_cut ? XZB_NEED_INPUT : XZB_DATA_ERROR; }
		const uint32_t b = *rc.cur++;
		if (i == 0 && b != 0x00) { rcp->in_pos = (uint32_t)(rc.cur - rcp->in); return XZB_DATA_ERROR; }
		rc.code = (rc.code << 8) | b;
	}
	rc.nb = rc.cur < rc.end ? (uint32_t)*rc.cur : 0u;
	uint32_t derr = 0;   // XZB_DATA_ERROR found by the LZ layer
	uint32_t state = d->state, rep0 = d->rep0, rep1 = d->rep1, rep2 = d->rep2, rep3 = d->rep3;
	uint32_t prev = pos != dict_start ? out[pos - 1] : 0;  // previous byte when prev_ok (none right after a reset)
	bool prev_ok = true;
	uint32_t pend_pos = 0, pend_len = 0, pend_val = 0;     // bytes out[pend_pos + lane], lane < pend_len, loaded but not stored yet
	while (pos < limit && !rc.err && !derr) {
		const uint32_t rel = pos - dict_start;  // dict.pos modulo 16 == bytes since dictionary reset modulo 16
		const uint32_t pos_state = rel & d->pos_mask;
		const uint32_t full = rel < dict_size_r ? rel : dict_size_r;
		// the byte a literal after a match is coded against: requested now if it is in memory, taken from the pending
		// copy's registers later (and only if this symbol is a literal)
		uint32_t match_byte = 0;
		const bool mb_wanted = state >= XZB_LIT_STATES && full > rep0;
		const uint32_t mb_pos = pos - rep0 - 1;
		const bool mb_pending = pend_len != 0 && mb_pos >= pend_pos;
		// (a prefetch, not a load: a load into a register that the next symbol overwrites would make every symbol wait
		// for the previous one's window read)
		if (mb_wanted && !mb_pending) asm volatile("prefetch.global.L1 [%0];" :: "l"(out + mb_pos));
		if (xzb_rcw_bit(rc, &d->is_match[state][pos_state]) == 0) {
			if (!prev_ok) prev = __shfl_sync(0xFFFFFFFFu, pend_val, pend_len - 1);   // a copy always ends at pos - 1
			if (mb_wanted) match_byte = mb_pending ? __shfl_sync(0xFFFFFFFFu, pend_val, mb_pos - pend_pos) : (uint32_t)out[mb_pos];
			xzb_prob *probs = d->literal + 3u * ((((rel << 8) + prev) & d->literal_mask) << d->lc);
			uint32_t symbol = 1;
			if (state < XZB_LIT_STATES) {
				state = state <= 3 ? 0 : state - 3;
				symbol = xzb_rcw_tree_walk(rc, probs, 8);
			} else {
				state = state <= 9 ? state - 3 : state - 6;
				uint32_t offset = 0x100;  // rc_matched_literal :270-300
				do {
					match_byte <<= 1;
					const uint32_t match_bit = match_byte & offset;
					const uint32_t bit = xzb_rcw_bit(rc, &probs[offset + match_bit + symbol]);
					symbol = (symbol << 1) | bit;
					offset &= bit ? match_bit : ~match_bit;
				} while (symbol < 0x100);
			}
			if (lane == 0) out[pos] = (uint8_t)symbol;
			prev = symbol & 0xFF; prev_ok = true;
			++pos;
			__syncwarp();
			continue;
		}
		uint32_t len;
		if (xzb_rcw_bit(rc, &d->is_rep[state]) == 0) {
			state = state < XZB_LIT_STATES ? 7 : 10;
			rep3 = rep2; rep2 = rep1; rep1 = rep0;
			len = xzb_rcw_len(rc, &d->match_len, pos_state);
			const uint32_t slot = xzb_rcw_tree_walk(rc, d->dist_slot[len < 6 ? len - 2 : 3], 6) - 64;
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
						const uint32_t bit = xzb_rcw_bit(rc, &probs[sym]);
						sym = (sym << 1) | bit;
						rep0 += bit ? off : 0u;
						off <<= 1;
					} while (--nbits > 0);
				} else {
					nbits -= XZB_ALIGN_BITS;
					do {  // rc_direct, range_decoder.h:375-388
						xzb_rcw_normalize(rc);
						rc.range >>= 1;
						rc.code -= rc.range;
						const uint32_t mask = 0u - (rc.code >> 31);
						rc.code += rc.range & mask;
						rep0 = (rep0 << 1) + (mask + 1);
					} while (--nbits > 0);
					rep0 <<= XZB_ALIGN_BITS;
					const uint32_t sym = xzb_rcw_tree_walk(rc, d->pos_align, XZB_ALIGN_BITS);  // rc_bittree_rev: first bit decoded is bit 0
					rep0 += ((sym >> 3) & 1) | ((sym >> 1) & 2) | ((sym << 1) & 4) | ((sym << 3) & 8);
					if (rep0 == 0xFFFFFFFFu) { derr = 2; break; }  // EOPM is not allowed in LZMA2 (this verdict also replaces "input ended")
				}
			}
			if (!(full > rep0)) { derr = 1; break; }
		} else {
			if (!(full > 0)) { derr = 1; break; }
			len = 0;
			if (xzb_rcw_bit(rc, &d->is_rep0[state]) == 0) {
				if (xzb_rcw_bit(rc, &d->is_rep0_long[state][pos_state]) == 0) {
					state = state < XZB_LIT_STATES ? 9 : 11;
					len = 1;   // short rep: a one-byte copy from rep0
				}
			} else {
				uint32_t dist;
				if (xzb_rcw_bit(rc, &d->is_rep1[state]) == 0) { dist = rep1; }
				else {
					if (xzb_rcw_bit(rc, &d->is_rep2[state]) == 0) { dist = rep2; }
					else { dist = rep3; rep3 = rep2; }
					rep2 = rep1;
				}
				rep1 = rep0; rep0 = dist;
			}
			if (len == 0) {
				state = state < XZB_LIT_STATES ? 8 : 11;
				len = xzb_rcw_len(rc, &d->rep_len, pos_state);
			}
			if (!(full > rep0)) { derr = 1; break; }
		}
		if (rc.err && len != 1) break;   // (a short rep is copied even when its last bit ran past the input, like a literal)
		// dict_repeat, lz_decoder.h:202-266; a match running past the chunk's size is corrupt
		if (len > limit - pos) { derr = 1; len = limit - pos; }
		// the previous copy goes to memory first: this one's source may lie in it
		if (pend_len != 0) {
			if (lane < pend_len) out[pend_pos + lane] = (uint8_t)pend_val;
			pend_len = 0;
			__syncwarp();
		}
		// overlapping copies are periodic with period rep0 + 1, so every byte has a source that was complete before
		// this match started
		const uint32_t back = pos - rep0 - 1, period = rep0 + 1;
		if (len <= 32) {
			uint32_t so = lane;
			if (period < 32) so = lane % period;   // (uniform branch: far matches, the common case, skip the division)
			if (lane < len) pend_val = out[back + so];
			pend_pos = pos; pend_len = len;
			prev_ok = false;
		} else {
			for (uint32_t i = lane; i < len; i += 32) out[pos + i] = out[back + (i < period ? i : i % period)];
			__syncwarp();
			prev = out[pos + len - 1]; prev_ok = true;
		}
		pos += len;
	}
	if (pend_len != 0) {
		if (lane < pend_len) out[pend_pos + lane] = (uint8_t)pend_val;
		__syncwarp();
	}
	d->state = state; d->rep0 = rep0; d->rep1 = rep1; d->rep2 = rep2; d->rep3 = rep3;
	*pos_ptr = pos;
	if (!rc.err && !derr) xzb_rcw_normalize(rc);  // lzma_decoder.c:661-690
	rcp->in_pos = (uint32_t)(rc.cur - rcp->in);
	if (derr == 2) return XZB_DATA_ERROR;
	if (rc.err) return chunk_cut ? XZB_NEED_INPUT : XZB_DATA_ERROR;
	if (derr) return XZB_DATA_ERROR;
	if (rc.code != 0) return XZB_DATA_ERROR;
	return XZB_OK;
}
