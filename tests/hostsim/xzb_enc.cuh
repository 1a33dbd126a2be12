// xzb_enc.cuh -- LZMA symbol selection + range coding + LZMA2 chunking for one .xz block, single-thread form.
// TEST HARNESS ONLY (tests/hostsim): the sequential statement of the encoder that the host simulation checks against
// the oracle; the product library contains the warp designs only (normal mode: xzb_parse_dp.cuh, fast mode and
// the coder both share: xzb_parse_warp.cuh).
//
// This is the strictly sequential half of the encoder (probabilities, price tables, reps and
// state all depend on every earlier symbol).  One CUDA block owns one .xz block; matches
// come from the match store filled by the parallel match-finder pass (xzb_mf.cuh), so
// "mf_find" here is a header + pair fetch and "mf_skip" is pointer arithmetic.
// Reference semantics per function are cited inline (paths relative to src/liblzma/).
#pragma once
#include "../../xz_b200/csrc/xzb_common.cuh"
#include "../../xz_b200/csrc/xzb_mf.cuh"

// ------------------------------------------------------------------------------------
// Match-store reader: stands in for lzma_mf (lz/lz_encoder.h:35-133) on the parser side.
// ------------------------------------------------------------------------------------
struct XzbMfView {
	const uint8_t *buf;
	uint32_t size;              // write_pos (whole block resident)
	uint32_t read_pos, read_ahead;
	uint32_t nice_len, stride;
	const uint32_t *mh;
	const xzb_pair *mp;
	const xzb_pair *ovf;
};

XZB_HD uint32_t xzb_mfv_avail(const XzbMfView &mf) { return mf.size - mf.read_pos; }

// lzma_mf_find (lz_encoder_mf.c:21-79): count, pairs and the (possibly extended) longest length.
XZB_HD uint32_t xzb_mfv_find(XzbMfView &mf, uint32_t *count_ptr, xzb_pair *matches)
{
	const uint32_t p = mf.read_pos;
	const uint32_t h = mf.mh[p];
	const uint32_t count = h & 0xFFFF;
	const xzb_pair *src = mf.mp + (size_t)p * mf.stride;
	if (count <= mf.stride) {
		for (uint32_t i = 0; i < count; ++i) matches[i] = src[i];
	} else {
		for (uint32_t i = 0; i + 1 < mf.stride; ++i) matches[i] = src[i];
		const xzb_pair *o = mf.ovf + src[mf.stride - 1].len;
		for (uint32_t i = mf.stride - 1; i < count; ++i) matches[i] = o[i - (mf.stride - 1)];
	}
	for (uint32_t i = 0; i < count; ++i) matches[i].len = XZB_PAIR_LEN(matches[i].len);  // drop the precomputed len2 / match byte
	*count_ptr = count;
	++mf.read_pos;
	++mf.read_ahead;
	return h >> 16;
}

// mf_skip (lz/lz_encoder.h:290-297): the insertions already happened in the match-finder pass.
XZB_HD void xzb_mfv_skip(XzbMfView &mf, uint32_t amount)
{
	mf.read_pos += amount;
	mf.read_ahead += amount;
}

// ------------------------------------------------------------------------------------
// Encoder state (lzma/lzma_encoder_private.h:38-150)
// ------------------------------------------------------------------------------------
struct XzbLenEnc {
	xzb_prob choice, choice2;
	xzb_prob low[XZB_POS_STATES_MAX][XZB_LEN_LOW], mid[XZB_POS_STATES_MAX][XZB_LEN_MID], high[XZB_LEN_HIGH];
	uint32_t prices[XZB_POS_STATES_MAX][XZB_LEN_SYMBOLS];
	uint32_t table_size;
	uint32_t counters[XZB_POS_STATES_MAX];
};

struct XzbOptimal {
	uint32_t state;
	uint8_t prev_1_is_literal, prev_2;
	uint32_t pos_prev_2, back_prev_2;
	uint32_t price, pos_prev, back_prev;
	uint32_t backs[XZB_REPS];
};

struct XzbRc {  // rangecoder/range_encoder.h:26-72
	uint64_t low, cache_size;
	uint32_t range;
	uint8_t cache;
	uint8_t *out;
	uint32_t out_pos;
};

struct XzbEnc {
	XzbRc rc;
	uint64_t uncomp_size;
	uint32_t state;
	uint32_t reps[XZB_REPS];
	xzb_pair matches[XZB_MATCH_LEN_MAX + 1];
	uint32_t matches_count, longest_match_length;
	uint32_t fast_mode, is_initialized;
	uint32_t pos_mask, lc, literal_mask;
	xzb_prob literal[16 * 0x300];
	xzb_prob is_match[XZB_STATES][XZB_POS_STATES_MAX];
	xzb_prob is_rep[XZB_STATES], is_rep0[XZB_STATES], is_rep1[XZB_STATES], is_rep2[XZB_STATES];
	xzb_prob is_rep0_long[XZB_STATES][XZB_POS_STATES_MAX];
	xzb_prob dist_slot[XZB_DIST_STATES][XZB_DIST_SLOTS];
	xzb_prob dist_special[XZB_FULL_DISTANCES - XZB_DIST_MODEL_END];
	xzb_prob dist_align[XZB_ALIGN_SIZE];
	XzbLenEnc match_len, rep_len;
	uint32_t dist_slot_prices[XZB_DIST_STATES][XZB_DIST_SLOTS];
	uint32_t dist_prices[XZB_DIST_STATES][XZB_FULL_DISTANCES];
	uint32_t dist_table_size, match_price_count;
	uint32_t align_prices[XZB_ALIGN_SIZE], align_price_count;
	uint32_t opts_end_index, opts_current_index;
	XzbOptimal opts[XZB_OPTS];
	uint8_t prices[128];   // rc price table copy
	XzbParams P;
	// statistics
	uint32_t n_symbols, n_chunks_lzma, n_chunks_raw;
};

// ---- range encoder: rangecoder/range_encoder.h.  The reference queues symbols and drains
// them in rc_encode() after each LZMA symbol; we encode immediately, and keep the one
// observable ordering effect explicit (see xzb_length_encode). ----
XZB_HD void xzb_rc_reset(XzbRc &rc) { rc.low = 0; rc.cache_size = 1; rc.range = 0xFFFFFFFFu; rc.cache = 0; }

XZB_HD void xzb_rc_shift_low(XzbRc &rc)  // :135-159
{
	if ((uint32_t)rc.low < 0xFF000000u || (uint32_t)(rc.low >> 32) != 0) {
		do {
			rc.out[rc.out_pos++] = (uint8_t)(rc.cache + (uint8_t)(rc.low >> 32));
			rc.cache = 0xFF;
		} while (--rc.cache_size != 0);
		rc.cache = (uint8_t)((rc.low >> 24) & 0xFF);
	}
	++rc.cache_size;
	rc.low = (rc.low & 0x00FFFFFF) << 8;
}

XZB_HD void xzb_rc_bit(XzbRc &rc, xzb_prob *prob, uint32_t bit)  // :78-84, :204-225
{
	if (rc.range < (1u << 24)) { xzb_rc_shift_low(rc); rc.range <<= 8; }
	xzb_prob p = *prob;
	const uint32_t bound = (rc.range >> 11) * p;
	if (bit == 0) { rc.range = bound; p += (2048 - p) >> 5; }
	else { rc.low += bound; rc.range -= bound; p -= p >> 5; }
	*prob = p;
}

XZB_HD void xzb_rc_bittree(XzbRc &rc, xzb_prob *probs, uint32_t bit_count, uint32_t symbol)  // :87-98
{
	uint32_t mi = 1;
	do {
		const uint32_t bit = (symbol >> --bit_count) & 1;
		xzb_rc_bit(rc, &probs[mi], bit);
		mi = (mi << 1) + bit;
	} while (bit_count != 0);
}

XZB_HD void xzb_rc_bittree_reverse(XzbRc &rc, xzb_prob *probs, uint32_t bit_count, uint32_t symbol)  // :101-113
{
	uint32_t mi = 1;
	do {
		const uint32_t bit = symbol & 1; symbol >>= 1;
		xzb_rc_bit(rc, &probs[mi], bit);
		mi = (mi << 1) + bit;
	} while (--bit_count != 0);
}

XZB_HD void xzb_rc_direct(XzbRc &rc, uint32_t value, uint32_t bit_count)  // :116-124, :227-234
{
	do {
		if (rc.range < (1u << 24)) { xzb_rc_shift_low(rc); rc.range <<= 8; }
		rc.range >>= 1;
		if ((value >> --bit_count) & 1) rc.low += rc.range;
	} while (bit_count != 0);
}

XZB_HD void xzb_rc_flush(XzbRc &rc)  // :127-132, :198-203, :236-249
{
	if (rc.range < (1u << 24)) { xzb_rc_shift_low(rc); rc.range <<= 8; }
	for (int i = 0; i < 5; ++i) xzb_rc_shift_low(rc);
	xzb_rc_reset(rc);
}

XZB_HD uint64_t xzb_rc_pending(const XzbRc &rc) { return rc.cache_size + 5 - 1; }  // :343-347

// ---- prices: rangecoder/price.h:28-90 ----
#define XZB_PR(e, idx) ((uint32_t)(e)->prices[(idx)])
XZB_HD uint32_t xzb_pr_bit(const XzbEnc *e, xzb_prob p, uint32_t bit) { return XZB_PR(e, (p ^ ((0u - bit) & 2047)) >> 4); }
XZB_HD uint32_t xzb_pr_bit0(const XzbEnc *e, xzb_prob p) { return XZB_PR(e, p >> 4); }
XZB_HD uint32_t xzb_pr_bit1(const XzbEnc *e, xzb_prob p) { return XZB_PR(e, (p ^ 2047) >> 4); }
XZB_HD uint32_t xzb_pr_bittree(const XzbEnc *e, const xzb_prob *probs, uint32_t levels, uint32_t symbol)
{
	uint32_t price = 0; symbol += 1u << levels;
	do { const uint32_t bit = symbol & 1; symbol >>= 1; price += xzb_pr_bit(e, probs[symbol], bit); } while (symbol != 1);
	return price;
}
XZB_HD uint32_t xzb_pr_bittree_reverse(const XzbEnc *e, const xzb_prob *probs, uint32_t levels, uint32_t symbol)
{
	uint32_t price = 0, mi = 1;
	do { const uint32_t bit = symbol & 1; symbol >>= 1; price += xzb_pr_bit(e, probs[mi], bit); mi = (mi << 1) + bit; } while (--levels != 0);
	return price;
}

// ---- state machine, lzma/lzma_common.h:55-114 ----
XZB_HD bool xzb_st_is_literal(uint32_t s) { return s < XZB_LIT_STATES; }
XZB_HD uint32_t xzb_st_literal(uint32_t s) { return s <= 3 ? 0 : (s <= 9 ? s - 3 : s - 6); }
XZB_HD uint32_t xzb_st_match(uint32_t s) { return s < XZB_LIT_STATES ? 7 : 10; }
XZB_HD uint32_t xzb_st_long_rep(uint32_t s) { return s < XZB_LIT_STATES ? 8 : 11; }
XZB_HD uint32_t xzb_st_short_rep(uint32_t s) { return s < XZB_LIT_STATES ? 9 : 11; }
XZB_HD xzb_prob *xzb_lit_subcoder(XzbEnc *e, uint32_t pos, uint32_t prev_byte)  // lzma_common.h:141-143
{
	return e->literal + 3u * ((((pos << 8) + prev_byte) & e->literal_mask) << e->lc);
}

// length_update_prices, lzma/lzma_encoder.c:76-102
XZB_HD_NOINLINE void xzb_length_update_prices(const XzbEnc *e, XzbLenEnc *lc, uint32_t pos_state)
{
	const uint32_t table_size = lc->table_size;
	lc->counters[pos_state] = table_size;
	const uint32_t a0 = xzb_pr_bit0(e, lc->choice), a1 = xzb_pr_bit1(e, lc->choice);
	const uint32_t b0 = a1 + xzb_pr_bit0(e, lc->choice2), b1 = a1 + xzb_pr_bit1(e, lc->choice2);
	uint32_t *prices = lc->prices[pos_state];
	uint32_t i;
	for (i = 0; i < table_size && i < XZB_LEN_LOW; ++i) prices[i] = a0 + xzb_pr_bittree(e, lc->low[pos_state], 3, i);
	for (; i < table_size && i < XZB_LEN_LOW + XZB_LEN_MID; ++i) prices[i] = b0 + xzb_pr_bittree(e, lc->mid[pos_state], 3, i - XZB_LEN_LOW);
	for (; i < table_size; ++i) prices[i] = b1 + xzb_pr_bittree(e, lc->high, 8, i - XZB_LEN_LOW - XZB_LEN_MID);
}

// length, lzma_encoder.c:105-134.  In the reference the bits are only queued here and hit the
// probabilities later (rc_encode), so a price refresh triggered by the counter still sees the
// probabilities from before this length's own bits: refresh first, then encode.
XZB_HD void xzb_length_encode(XzbEnc *e, XzbLenEnc *lc, uint32_t pos_state, uint32_t len)
{
	XzbRc &rc = e->rc;
	if (!e->fast_mode)
		if (--lc->counters[pos_state] == 0)
			xzb_length_update_prices(e, lc, pos_state);
	len -= XZB_MATCH_LEN_MIN;
	if (len < XZB_LEN_LOW) {
		xzb_rc_bit(rc, &lc->choice, 0);
		xzb_rc_bittree(rc, lc->low[pos_state], 3, len);
	} else {
		xzb_rc_bit(rc, &lc->choice, 1);
		len -= XZB_LEN_LOW;
		if (len < XZB_LEN_MID) {
			xzb_rc_bit(rc, &lc->choice2, 0);
			xzb_rc_bittree(rc, lc->mid[pos_state], 3, len);
		} else {
			xzb_rc_bit(rc, &lc->choice2, 1);
			len -= XZB_LEN_MID;
			xzb_rc_bittree(rc, lc->high, 8, len);
		}
	}
}

XZB_HD_NOINLINE void xzb_len_reset(const XzbEnc *e, XzbLenEnc *lc, uint32_t num_pos_states, uint32_t fast_mode)  // lzma_encoder.c:505-525
{
	lc->choice = 1024; lc->choice2 = 1024;
	for (uint32_t ps = 0; ps < num_pos_states; ++ps) {
		for (int i = 0; i < XZB_LEN_LOW; ++i) lc->low[ps][i] = 1024;
		for (int i = 0; i < XZB_LEN_MID; ++i) lc->mid[ps][i] = 1024;
	}
	for (int i = 0; i < XZB_LEN_HIGH; ++i) lc->high[i] = 1024;
	if (!fast_mode)
		for (uint32_t ps = 0; ps < num_pos_states; ++ps) xzb_length_update_prices(e, lc, ps);
}

// lzma_lzma_encoder_reset, lzma_encoder.c:528-598
XZB_HD_NOINLINE void xzb_enc_reset(XzbEnc *e)
{
	const XzbParams &o = e->P;
	e->pos_mask = (1u << o.pb) - 1;
	e->lc = o.lc;
	e->literal_mask = (0x100u << o.lp) - (0x100u >> o.lc);
	xzb_rc_reset(e->rc);
	e->state = 0;
	for (int i = 0; i < XZB_REPS; ++i) e->reps[i] = 0;
	const uint32_t coders = 0x300u << (o.lc + o.lp);
	for (uint32_t i = 0; i < coders; ++i) e->literal[i] = 1024;
	for (int i = 0; i < XZB_STATES; ++i) {
		for (uint32_t j = 0; j <= e->pos_mask; ++j) { e->is_match[i][j] = 1024; e->is_rep0_long[i][j] = 1024; }
		e->is_rep[i] = e->is_rep0[i] = e->is_rep1[i] = e->is_rep2[i] = 1024;
	}
	for (int i = 0; i < XZB_FULL_DISTANCES - XZB_DIST_MODEL_END; ++i) e->dist_special[i] = 1024;
	for (int i = 0; i < XZB_DIST_STATES; ++i) for (int j = 0; j < XZB_DIST_SLOTS; ++j) e->dist_slot[i][j] = 1024;
	for (int i = 0; i < XZB_ALIGN_SIZE; ++i) e->dist_align[i] = 1024;
	xzb_len_reset(e, &e->match_len, 1u << o.pb, e->fast_mode);
	xzb_len_reset(e, &e->rep_len, 1u << o.pb, e->fast_mode);
	e->match_price_count = 0xFFFFFFFFu / 2;
	e->align_price_count = 0xFFFFFFFFu / 2;
	e->opts_end_index = 0; e->opts_current_index = 0;
}

// lzma_lzma_encoder_create, lzma_encoder.c:601-707 (options were validated on the host)
XZB_HD_NOINLINE void xzb_enc_create(XzbEnc *e, const XzbParams &P, const uint8_t *price_table)
{
	e->P = P;
	for (int i = 0; i < 128; ++i) e->prices[i] = price_table[i];
	e->fast_mode = P.mode == XZB_MODE_FAST;
	e->dist_table_size = P.dist_table_size;
	e->match_len.table_size = P.len_table_size;
	e->rep_len.table_size = P.len_table_size;
	e->is_initialized = 0;
	e->uncomp_size = 0;
	e->n_symbols = 0; e->n_chunks_lzma = 0; e->n_chunks_raw = 0;
	xzb_enc_reset(e);
}

// literal_matched :22-43, literal :46-69
XZB_HD void xzb_literal_encode(XzbEnc *e, const XzbMfView &mf, uint32_t position)
{
	const uint8_t cur_byte = mf.buf[mf.read_pos - mf.read_ahead];
	xzb_prob *sub = xzb_lit_subcoder(e, position, mf.buf[mf.read_pos - mf.read_ahead - 1]);
	if (xzb_st_is_literal(e->state)) {
		e->state = e->state <= 3 ? 0 : e->state - 3;
		xzb_rc_bittree(e->rc, sub, 8, cur_byte);
	} else {
		e->state = e->state <= 9 ? e->state - 3 : e->state - 6;
		uint32_t match_byte = mf.buf[mf.read_pos - e->reps[0] - 1 - mf.read_ahead];
		uint32_t offset = 0x100, symbol = cur_byte + (1u << 8);
		do {
			match_byte <<= 1;
			const uint32_t match_bit = match_byte & offset;
			const uint32_t idx = offset + match_bit + (symbol >> 8);
			const uint32_t bit = (symbol >> 7) & 1;
			xzb_rc_bit(e->rc, &sub[idx], bit);
			symbol <<= 1;
			offset &= ~(match_byte ^ symbol);
		} while (symbol < (1u << 16));
	}
}

// match, lzma_encoder.c:141-181
XZB_HD void xzb_match_encode(XzbEnc *e, uint32_t pos_state, uint32_t distance, uint32_t len)
{
	e->state = xzb_st_match(e->state);
	xzb_length_encode(e, &e->match_len, pos_state, len);
	const uint32_t slot = xzb_dist_slot(distance);
	xzb_rc_bittree(e->rc, e->dist_slot[xzb_dist_state(len)], 6, slot);
	if (slot >= XZB_DIST_MODEL_START) {
		const uint32_t footer_bits = (slot >> 1) - 1;
		const uint32_t base = (2 | (slot & 1)) << footer_bits;
		const uint32_t reduced = distance - base;
		if (slot < XZB_DIST_MODEL_END) {
			xzb_rc_bittree_reverse(e->rc, e->dist_special + base - slot - 1, footer_bits, reduced);
		} else {
			xzb_rc_direct(e->rc, reduced >> XZB_ALIGN_BITS, footer_bits - XZB_ALIGN_BITS);
			xzb_rc_bittree_reverse(e->rc, e->dist_align, XZB_ALIGN_BITS, reduced & XZB_ALIGN_MASK);
			++e->align_price_count;
		}
	}
	e->reps[3] = e->reps[2]; e->reps[2] = e->reps[1]; e->reps[1] = e->reps[0]; e->reps[0] = distance;
	++e->match_price_count;
}

// rep_match, lzma_encoder.c:188-225
XZB_HD void xzb_rep_match_encode(XzbEnc *e, uint32_t pos_state, uint32_t rep, uint32_t len)
{
	XzbRc &rc = e->rc;
	if (rep == 0) {
		xzb_rc_bit(rc, &e->is_rep0[e->state], 0);
		xzb_rc_bit(rc, &e->is_rep0_long[e->state][pos_state], len != 1);
	} else {
		const uint32_t distance = e->reps[rep];
		xzb_rc_bit(rc, &e->is_rep0[e->state], 1);
		if (rep == 1) {
			xzb_rc_bit(rc, &e->is_rep1[e->state], 0);
		} else {
			xzb_rc_bit(rc, &e->is_rep1[e->state], 1);
			xzb_rc_bit(rc, &e->is_rep2[e->state], rep - 2);
			if (rep == 3) e->reps[3] = e->reps[2];
			e->reps[2] = e->reps[1];
		}
		e->reps[1] = e->reps[0];
		e->reps[0] = distance;
	}
	if (len == 1) {
		e->state = xzb_st_short_rep(e->state);
	} else {
		xzb_length_encode(e, &e->rep_len, pos_state, len);
		e->state = xzb_st_long_rep(e->state);
	}
}

// encode_symbol, lzma_encoder.c:232-263
XZB_HD void xzb_encode_symbol(XzbEnc *e, XzbMfView &mf, uint32_t back, uint32_t len, uint32_t position)
{
	const uint32_t pos_state = position & e->pos_mask;
	++e->n_symbols;
	if (back == XZB_BACK_LITERAL) {
		xzb_rc_bit(e->rc, &e->is_match[e->state][pos_state], 0);
		xzb_literal_encode(e, mf, position);
	} else {
		xzb_rc_bit(e->rc, &e->is_match[e->state][pos_state], 1);
		if (back < XZB_REPS) {
			xzb_rc_bit(e->rc, &e->is_rep[e->state], 1);
			xzb_rep_match_encode(e, pos_state, back, len);
		} else {
			xzb_rc_bit(e->rc, &e->is_rep[e->state], 0);
			xzb_match_encode(e, pos_state, back - XZB_REPS, len);
		}
	}
	mf.read_ahead -= len;
}

// ------------------------------------------------------------------------------------
// lzma_lzma_optimum_fast, lzma/lzma_encoder_optimum_fast.c:19-169
// ------------------------------------------------------------------------------------
XZB_HD bool xzb_change_pair(uint32_t small_dist, uint32_t big_dist) { return (big_dist >> 7) > small_dist; }
XZB_HD bool xzb_ne16(const uint8_t *a, const uint8_t *b) { return a[0] != b[0] || a[1] != b[1]; }

XZB_HD_NOINLINE void xzb_optimum_fast(XzbEnc *e, XzbMfView &mf, uint32_t *back_res, uint32_t *len_res)
{
	const uint32_t nice_len = mf.nice_len;
	uint32_t len_main, matches_count;
	if (mf.read_ahead == 0) {
		len_main = xzb_mfv_find(mf, &matches_count, e->matches);
	} else {
		len_main = e->longest_match_length;
		matches_count = e->matches_count;
	}
	const uint8_t *buf = mf.buf + mf.read_pos - 1;
	const uint32_t buf_avail = xzb_min(xzb_mfv_avail(mf) + 1, XZB_MATCH_LEN_MAX);
	if (buf_avail < 2) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return; }

	uint32_t rep_len = 0, rep_index = 0;
	for (uint32_t i = 0; i < XZB_REPS; ++i) {
		const uint8_t *bb = buf - e->reps[i] - 1;
		if (xzb_ne16(buf, bb)) continue;
		const uint32_t len = xzb_memcmplen(buf, bb, 2, buf_avail);
		if (len >= nice_len) { *back_res = i; *len_res = len; xzb_mfv_skip(mf, len - 1); return; }
		if (len > rep_len) { rep_index = i; rep_len = len; }
	}
	if (len_main >= nice_len) {
		*back_res = e->matches[matches_count - 1].dist + XZB_REPS; *len_res = len_main;
		xzb_mfv_skip(mf, len_main - 1); return;
	}
	uint32_t back_main = 0;
	if (len_main >= 2) {
		back_main = e->matches[matches_count - 1].dist;
		while (matches_count > 1 && len_main == e->matches[matches_count - 2].len + 1) {
			if (!xzb_change_pair(e->matches[matches_count - 2].dist, back_main)) break;
			--matches_count;
			len_main = e->matches[matches_count - 1].len;
			back_main = e->matches[matches_count - 1].dist;
		}
		if (len_main == 2 && back_main >= 0x80) len_main = 1;
	}
	if (rep_len >= 2) {
		if (rep_len + 1 >= len_main
				|| (rep_len + 2 >= len_main && back_main > (1u << 9))
				|| (rep_len + 3 >= len_main && back_main > (1u << 15))) {
			*back_res = rep_index; *len_res = rep_len; xzb_mfv_skip(mf, rep_len - 1); return;
		}
	}
	if (len_main < 2 || buf_avail <= 2) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return; }

	e->longest_match_length = xzb_mfv_find(mf, &e->matches_count, e->matches);
	if (e->longest_match_length >= 2) {
		const uint32_t new_dist = e->matches[e->matches_count - 1].dist;
		if ((e->longest_match_length >= len_main && new_dist < back_main)
				|| (e->longest_match_length == len_main + 1 && !xzb_change_pair(back_main, new_dist))
				|| (e->longest_match_length > len_main + 1)
				|| (e->longest_match_length + 1 >= len_main && len_main >= 3 && xzb_change_pair(new_dist, back_main))) {
			*back_res = XZB_BACK_LITERAL; *len_res = 1; return;
		}
	}
	++buf;
	const uint32_t limit = xzb_max(2, len_main - 1);
	for (uint32_t i = 0; i < XZB_REPS; ++i) {
		const uint8_t *bb = buf - e->reps[i] - 1;
		if (xzb_memcmplen(buf, bb, 0, limit) == limit) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return; }  // memcmp(...) == 0
	}
	*back_res = back_main + XZB_REPS; *len_res = len_main;
	xzb_mfv_skip(mf, len_main - 2);
}

// ------------------------------------------------------------------------------------
// lzma_lzma_optimum_normal, lzma/lzma_encoder_optimum_normal.c
// ------------------------------------------------------------------------------------
XZB_HD uint32_t xzb_literal_price(XzbEnc *e, uint32_t pos, uint32_t prev_byte, bool match_mode, uint32_t match_byte, uint32_t symbol)  // :20-53
{
	const xzb_prob *sub = xzb_lit_subcoder(e, pos, prev_byte);
	uint32_t price = 0;
	if (!match_mode) {
		price = xzb_pr_bittree(e, sub, 8, symbol);
	} else {
		uint32_t offset = 0x100; symbol += 1u << 8;
		do {
			match_byte <<= 1;
			const uint32_t match_bit = match_byte & offset;
			const uint32_t idx = offset + match_bit + (symbol >> 8);
			const uint32_t bit = (symbol >> 7) & 1;
			price += xzb_pr_bit(e, sub[idx], bit);
			symbol <<= 1;
			offset &= ~(match_byte ^ symbol);
		} while (symbol < (1u << 16));
	}
	return price;
}
XZB_HD uint32_t xzb_len_price(const XzbLenEnc *l, uint32_t len, uint32_t ps) { return l->prices[ps][len - XZB_MATCH_LEN_MIN]; }  // :56-63
XZB_HD uint32_t xzb_short_rep_price(const XzbEnc *e, uint32_t st, uint32_t ps) { return xzb_pr_bit0(e, e->is_rep0[st]) + xzb_pr_bit0(e, e->is_rep0_long[st][ps]); }  // :66-72
XZB_HD uint32_t xzb_pure_rep_price(const XzbEnc *e, uint32_t rep, uint32_t st, uint32_t ps)  // :75-97
{
	uint32_t price;
	if (rep == 0) {
		price = xzb_pr_bit0(e, e->is_rep0[st]) + xzb_pr_bit1(e, e->is_rep0_long[st][ps]);
	} else {
		price = xzb_pr_bit1(e, e->is_rep0[st]);
		if (rep == 1) price += xzb_pr_bit0(e, e->is_rep1[st]);
		else { price += xzb_pr_bit1(e, e->is_rep1[st]); price += xzb_pr_bit(e, e->is_rep2[st], rep - 2); }
	}
	return price;
}
XZB_HD uint32_t xzb_rep_price(const XzbEnc *e, uint32_t rep, uint32_t len, uint32_t st, uint32_t ps) { return xzb_len_price(&e->rep_len, len, ps) + xzb_pure_rep_price(e, rep, st, ps); }  // :100-107
XZB_HD uint32_t xzb_dist_len_price(const XzbEnc *e, uint32_t dist, uint32_t len, uint32_t ps)  // :110-128
{
	const uint32_t ds = xzb_dist_state(len);
	uint32_t price;
	if (dist < XZB_FULL_DISTANCES) price = e->dist_prices[ds][dist];
	else price = e->dist_slot_prices[ds][xzb_dist_slot(dist)] + e->align_prices[dist & XZB_ALIGN_MASK];
	return price + xzb_len_price(&e->match_len, len, ps);
}
XZB_HD_NOINLINE void xzb_fill_dist_prices(XzbEnc *e)  // :131-183
{
	for (uint32_t ds = 0; ds < XZB_DIST_STATES; ++ds) {
		uint32_t *sp = e->dist_slot_prices[ds];
		for (uint32_t s = 0; s < e->dist_table_size; ++s) sp[s] = xzb_pr_bittree(e, e->dist_slot[ds], 6, s);
		for (uint32_t s = XZB_DIST_MODEL_END; s < e->dist_table_size; ++s) sp[s] += (((s >> 1) - 1) - XZB_ALIGN_BITS) << 4;
		for (uint32_t i = 0; i < XZB_DIST_MODEL_START; ++i) e->dist_prices[ds][i] = sp[i];
	}
	for (uint32_t i = XZB_DIST_MODEL_START; i < XZB_FULL_DISTANCES; ++i) {
		const uint32_t slot = xzb_dist_slot(i);
		const uint32_t footer_bits = (slot >> 1) - 1;
		const uint32_t base = (2 | (slot & 1)) << footer_bits;
		const uint32_t price = xzb_pr_bittree_reverse(e, e->dist_special + base - slot - 1, footer_bits, i - base);
		for (uint32_t ds = 0; ds < XZB_DIST_STATES; ++ds) e->dist_prices[ds][i] = price + e->dist_slot_prices[ds][slot];
	}
	e->match_price_count = 0;
}
XZB_HD_NOINLINE void xzb_fill_align_prices(XzbEnc *e)  // :186-195
{
	for (uint32_t i = 0; i < XZB_ALIGN_SIZE; ++i) e->align_prices[i] = xzb_pr_bittree_reverse(e, e->dist_align, XZB_ALIGN_BITS, i);
	e->align_price_count = 0;
}

XZB_HD void xzb_make_literal(XzbOptimal *o) { o->back_prev = XZB_BACK_LITERAL; o->prev_1_is_literal = 0; }
XZB_HD void xzb_make_short_rep(XzbOptimal *o) { o->back_prev = 0; o->prev_1_is_literal = 0; }

XZB_HD_NOINLINE void xzb_backward(XzbEnc *e, uint32_t *len_res, uint32_t *back_res, uint32_t cur)  // :222-263
{
	XzbOptimal *opts = e->opts;
	e->opts_end_index = cur;
	uint32_t pos_mem = opts[cur].pos_prev;
	uint32_t back_mem = opts[cur].back_prev;
	do {
		if (opts[cur].prev_1_is_literal) {
			xzb_make_literal(&opts[pos_mem]);
			opts[pos_mem].pos_prev = pos_mem - 1;
			if (opts[cur].prev_2) {
				opts[pos_mem - 1].prev_1_is_literal = 0;
				opts[pos_mem - 1].pos_prev = opts[cur].pos_prev_2;
				opts[pos_mem - 1].back_prev = opts[cur].back_prev_2;
			}
		}
		const uint32_t pos_prev = pos_mem, back_cur = back_mem;
		back_mem = opts[pos_prev].back_prev;
		pos_mem = opts[pos_prev].pos_prev;
		opts[pos_prev].back_prev = back_cur;
		opts[pos_prev].pos_prev = cur;
		cur = pos_prev;
	} while (cur != 0);
	e->opts_current_index = opts[0].pos_prev;
	*len_res = opts[0].pos_prev;
	*back_res = opts[0].back_prev;
}

XZB_HD_NOINLINE uint32_t xzb_helper1(XzbEnc *e, XzbMfView &mf, uint32_t *back_res, uint32_t *len_res, uint32_t position)  // :270-439
{
	XzbOptimal *opts = e->opts;
	const uint32_t nice_len = mf.nice_len;
	uint32_t len_main, matches_count;
	if (mf.read_ahead == 0) {
		len_main = xzb_mfv_find(mf, &matches_count, e->matches);
	} else {
		len_main = e->longest_match_length;
		matches_count = e->matches_count;
	}
	const uint32_t buf_avail = xzb_min(xzb_mfv_avail(mf) + 1, XZB_MATCH_LEN_MAX);
	if (buf_avail < 2) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return 0xFFFFFFFFu; }
	const uint8_t *buf = mf.buf + mf.read_pos - 1;

	uint32_t rep_lens[XZB_REPS];
	uint32_t rep_max_index = 0;
	for (uint32_t i = 0; i < XZB_REPS; ++i) {
		const uint8_t *bb = buf - e->reps[i] - 1;
		if (xzb_ne16(buf, bb)) { rep_lens[i] = 0; continue; }
		rep_lens[i] = xzb_memcmplen(buf, bb, 2, buf_avail);
		if (rep_lens[i] > rep_lens[rep_max_index]) rep_max_index = i;
	}
	if (rep_lens[rep_max_index] >= nice_len) {
		*back_res = rep_max_index; *len_res = rep_lens[rep_max_index];
		xzb_mfv_skip(mf, *len_res - 1); return 0xFFFFFFFFu;
	}
	if (len_main >= nice_len) {
		*back_res = e->matches[matches_count - 1].dist + XZB_REPS; *len_res = len_main;
		xzb_mfv_skip(mf, len_main - 1); return 0xFFFFFFFFu;
	}
	const uint8_t current_byte = *buf;
	const uint8_t match_byte = *(buf - e->reps[0] - 1);
	if (len_main < 2 && current_byte != match_byte && rep_lens[rep_max_index] < 2) {
		*back_res = XZB_BACK_LITERAL; *len_res = 1; return 0xFFFFFFFFu;
	}
	opts[0].state = e->state;
	const uint32_t pos_state = position & e->pos_mask;
	opts[1].price = xzb_pr_bit0(e, e->is_match[e->state][pos_state])
			+ xzb_literal_price(e, position, buf[-1], !xzb_st_is_literal(e->state), match_byte, current_byte);
	xzb_make_literal(&opts[1]);
	const uint32_t match_price = xzb_pr_bit1(e, e->is_match[e->state][pos_state]);
	const uint32_t rep_match_price = match_price + xzb_pr_bit1(e, e->is_rep[e->state]);
	if (match_byte == current_byte) {
		const uint32_t srp = rep_match_price + xzb_short_rep_price(e, e->state, pos_state);
		if (srp < opts[1].price) { opts[1].price = srp; xzb_make_short_rep(&opts[1]); }
	}
	const uint32_t len_end = xzb_max(len_main, rep_lens[rep_max_index]);
	if (len_end < 2) { *back_res = opts[1].back_prev; *len_res = 1; return 0xFFFFFFFFu; }
	opts[1].pos_prev = 0;
	for (uint32_t i = 0; i < XZB_REPS; ++i) opts[0].backs[i] = e->reps[i];
	uint32_t len = len_end;
	do { opts[len].price = XZB_INFINITY_PRICE; } while (--len >= 2);

	for (uint32_t i = 0; i < XZB_REPS; ++i) {
		uint32_t rep_len = rep_lens[i];
		if (rep_len < 2) continue;
		const uint32_t price = rep_match_price + xzb_pure_rep_price(e, i, e->state, pos_state);
		do {
			const uint32_t p = price + xzb_len_price(&e->rep_len, rep_len, pos_state);
			if (p < opts[rep_len].price) {
				opts[rep_len].price = p; opts[rep_len].pos_prev = 0;
				opts[rep_len].back_prev = i; opts[rep_len].prev_1_is_literal = 0;
			}
		} while (--rep_len >= 2);
	}
	const uint32_t normal_match_price = match_price + xzb_pr_bit0(e, e->is_rep[e->state]);
	len = rep_lens[0] >= 2 ? rep_lens[0] + 1 : 2;
	if (len <= len_main) {
		uint32_t i = 0;
		while (len > e->matches[i].len) ++i;
		for (;; ++len) {
			const uint32_t dist = e->matches[i].dist;
			const uint32_t p = normal_match_price + xzb_dist_len_price(e, dist, len, pos_state);
			if (p < opts[len].price) {
				opts[len].price = p; opts[len].pos_prev = 0;
				opts[len].back_prev = dist + XZB_REPS; opts[len].prev_1_is_literal = 0;
			}
			if (len == e->matches[i].len)
				if (++i == matches_count) break;
		}
	}
	return len_end;
}

XZB_HD_NOINLINE uint32_t xzb_helper2(XzbEnc *e, uint32_t *reps, const uint8_t *buf, uint32_t len_end,
		uint32_t position, const uint32_t cur, const uint32_t nice_len, const uint32_t buf_avail_full)  // :442-799
{
	XzbOptimal *opts = e->opts;
	uint32_t matches_count = e->matches_count;
	uint32_t new_len = e->longest_match_length;
	uint32_t pos_prev = opts[cur].pos_prev;
	uint32_t state;

	if (opts[cur].prev_1_is_literal) {
		--pos_prev;
		if (opts[cur].prev_2) {
			state = opts[opts[cur].pos_prev_2].state;
			if (opts[cur].back_prev_2 < XZB_REPS) state = xzb_st_long_rep(state);
			else state = xzb_st_match(state);
		} else {
			state = opts[pos_prev].state;
		}
		state = xzb_st_literal(state);
	} else {
		state = opts[pos_prev].state;
	}

	if (pos_prev == cur - 1) {
		if (opts[cur].back_prev == 0) state = xzb_st_short_rep(state);
		else state = xzb_st_literal(state);
	} else {
		uint32_t pos;
		if (opts[cur].prev_1_is_literal && opts[cur].prev_2) {
			pos_prev = opts[cur].pos_prev_2;
			pos = opts[cur].back_prev_2;
			state = xzb_st_long_rep(state);
		} else {
			pos = opts[cur].back_prev;
			if (pos < XZB_REPS) state = xzb_st_long_rep(state);
			else state = xzb_st_match(state);
		}
		if (pos < XZB_REPS) {
			reps[0] = opts[pos_prev].backs[pos];
			uint32_t i;
			for (i = 1; i <= pos; ++i) reps[i] = opts[pos_prev].backs[i - 1];
			for (; i < XZB_REPS; ++i) reps[i] = opts[pos_prev].backs[i];
		} else {
			reps[0] = pos - XZB_REPS;
			for (uint32_t i = 1; i < XZB_REPS; ++i) reps[i] = opts[pos_prev].backs[i - 1];
		}
	}
	opts[cur].state = state;
	for (uint32_t i = 0; i < XZB_REPS; ++i) opts[cur].backs[i] = reps[i];

	const uint32_t cur_price = opts[cur].price;
	const uint8_t current_byte = *buf;
	const uint8_t match_byte = *(buf - reps[0] - 1);
	const uint32_t pos_state = position & e->pos_mask;
	const uint32_t cur_and_1_price = cur_price + xzb_pr_bit0(e, e->is_match[state][pos_state])
			+ xzb_literal_price(e, position, buf[-1], !xzb_st_is_literal(state), match_byte, current_byte);
	bool next_is_literal = false;
	if (cur_and_1_price < opts[cur + 1].price) {
		opts[cur + 1].price = cur_and_1_price;
		opts[cur + 1].pos_prev = cur;
		xzb_make_literal(&opts[cur + 1]);
		next_is_literal = true;
	}
	const uint32_t match_price = cur_price + xzb_pr_bit1(e, e->is_match[state][pos_state]);
	const uint32_t rep_match_price = match_price + xzb_pr_bit1(e, e->is_rep[state]);
	if (match_byte == current_byte && !(opts[cur + 1].pos_prev < cur && opts[cur + 1].back_prev == 0)) {
		const uint32_t srp = rep_match_price + xzb_short_rep_price(e, state, pos_state);
		if (srp <= opts[cur + 1].price) {
			opts[cur + 1].price = srp;
			opts[cur + 1].pos_prev = cur;
			xzb_make_short_rep(&opts[cur + 1]);
			next_is_literal = true;
		}
	}
	if (buf_avail_full < 2) return len_end;
	const uint32_t buf_avail = xzb_min(buf_avail_full, nice_len);

	if (!next_is_literal && match_byte != current_byte) {
		// literal + rep0, :562-597
		const uint8_t *bb = buf - reps[0] - 1;
		const uint32_t limit = xzb_min(buf_avail_full, nice_len + 1);
		const uint32_t len_test = xzb_memcmplen(buf, bb, 1, limit) - 1;
		if (len_test >= 2) {
			const uint32_t state_2 = xzb_st_literal(state);
			const uint32_t psn = (position + 1) & e->pos_mask;
			const uint32_t nrmp = cur_and_1_price + xzb_pr_bit1(e, e->is_match[state_2][psn]) + xzb_pr_bit1(e, e->is_rep[state_2]);
			const uint32_t offset = cur + 1 + len_test;
			while (len_end < offset) opts[++len_end].price = XZB_INFINITY_PRICE;
			const uint32_t p = nrmp + xzb_rep_price(e, 0, len_test, state_2, psn);
			if (p < opts[offset].price) {
				opts[offset].price = p; opts[offset].pos_prev = cur + 1; opts[offset].back_prev = 0;
				opts[offset].prev_1_is_literal = 1; opts[offset].prev_2 = 0;
			}
		}
	}

	uint32_t start_len = 2;
	for (uint32_t rep_index = 0; rep_index < XZB_REPS; ++rep_index) {
		const uint8_t *bb = buf - reps[rep_index] - 1;
		if (xzb_ne16(buf, bb)) continue;
		uint32_t len_test = xzb_memcmplen(buf, bb, 2, buf_avail);
		while (len_end < cur + len_test) opts[++len_end].price = XZB_INFINITY_PRICE;
		const uint32_t len_test_temp = len_test;
		const uint32_t price = rep_match_price + xzb_pure_rep_price(e, rep_index, state, pos_state);
		do {
			const uint32_t p = price + xzb_len_price(&e->rep_len, len_test, pos_state);
			if (p < opts[cur + len_test].price) {
				opts[cur + len_test].price = p; opts[cur + len_test].pos_prev = cur;
				opts[cur + len_test].back_prev = rep_index; opts[cur + len_test].prev_1_is_literal = 0;
			}
		} while (--len_test >= 2);
		len_test = len_test_temp;
		if (rep_index == 0) start_len = len_test + 1;

		uint32_t len_test_2 = len_test + 1;
		const uint32_t limit = xzb_min(buf_avail_full, len_test_2 + nice_len);
		if (len_test_2 < limit) len_test_2 = xzb_memcmplen(buf, bb, len_test_2, limit);
		len_test_2 -= len_test + 1;
		if (len_test_2 >= 2) {
			uint32_t state_2 = xzb_st_long_rep(state);
			uint32_t psn = (position + len_test) & e->pos_mask;
			const uint32_t calp = price + xzb_len_price(&e->rep_len, len_test, pos_state)
					+ xzb_pr_bit0(e, e->is_match[state_2][psn])
					+ xzb_literal_price(e, position + len_test, buf[len_test - 1], true, bb[len_test], buf[len_test]);
			state_2 = xzb_st_literal(state_2);
			psn = (position + len_test + 1) & e->pos_mask;
			const uint32_t nrmp = calp + xzb_pr_bit1(e, e->is_match[state_2][psn]) + xzb_pr_bit1(e, e->is_rep[state_2]);
			const uint32_t offset = cur + len_test + 1 + len_test_2;
			while (len_end < offset) opts[++len_end].price = XZB_INFINITY_PRICE;
			const uint32_t p = nrmp + xzb_rep_price(e, 0, len_test_2, state_2, psn);
			if (p < opts[offset].price) {
				opts[offset].price = p; opts[offset].pos_prev = cur + len_test + 1; opts[offset].back_prev = 0;
				opts[offset].prev_1_is_literal = 1; opts[offset].prev_2 = 1;
				opts[offset].pos_prev_2 = cur; opts[offset].back_prev_2 = rep_index;
			}
		}
	}

	if (new_len > buf_avail) {
		new_len = buf_avail;
		matches_count = 0;
		while (new_len > e->matches[matches_count].len) ++matches_count;
		e->matches[matches_count++].len = new_len;
	}
	if (new_len >= start_len) {
		const uint32_t normal_match_price = match_price + xzb_pr_bit0(e, e->is_rep[state]);
		while (len_end < cur + new_len) opts[++len_end].price = XZB_INFINITY_PRICE;
		uint32_t i = 0;
		while (start_len > e->matches[i].len) ++i;
		for (uint32_t len_test = start_len;; ++len_test) {
			const uint32_t cur_back = e->matches[i].dist;
			uint32_t p = normal_match_price + xzb_dist_len_price(e, cur_back, len_test, pos_state);
			if (p < opts[cur + len_test].price) {
				opts[cur + len_test].price = p; opts[cur + len_test].pos_prev = cur;
				opts[cur + len_test].back_prev = cur_back + XZB_REPS; opts[cur + len_test].prev_1_is_literal = 0;
			}
			if (len_test == e->matches[i].len) {
				// match + literal + rep0, :729-790
				const uint8_t *bb = buf - cur_back - 1;
				uint32_t len_test_2 = len_test + 1;
				const uint32_t limit = xzb_min(buf_avail_full, len_test_2 + nice_len);
				if (len_test_2 < limit) len_test_2 = xzb_memcmplen(buf, bb, len_test_2, limit);
				len_test_2 -= len_test + 1;
				if (len_test_2 >= 2) {
					uint32_t state_2 = xzb_st_match(state);
					uint32_t psn = (position + len_test) & e->pos_mask;
					const uint32_t calp = p + xzb_pr_bit0(e, e->is_match[state_2][psn])
							+ xzb_literal_price(e, position + len_test, buf[len_test - 1], true, bb[len_test], buf[len_test]);
					state_2 = xzb_st_literal(state_2);
					psn = (psn + 1) & e->pos_mask;
					const uint32_t nrmp = calp + xzb_pr_bit1(e, e->is_match[state_2][psn]) + xzb_pr_bit1(e, e->is_rep[state_2]);
					const uint32_t offset = cur + len_test + 1 + len_test_2;
					while (len_end < offset) opts[++len_end].price = XZB_INFINITY_PRICE;
					p = nrmp + xzb_rep_price(e, 0, len_test_2, state_2, psn);
					if (p < opts[offset].price) {
						opts[offset].price = p; opts[offset].pos_prev = cur + len_test + 1; opts[offset].back_prev = 0;
						opts[offset].prev_1_is_literal = 1; opts[offset].prev_2 = 1;
						opts[offset].pos_prev_2 = cur; opts[offset].back_prev_2 = cur_back + XZB_REPS;
					}
				}
				if (++i == matches_count) break;
			}
		}
	}
	return len_end;
}

XZB_HD_NOINLINE void xzb_optimum_normal(XzbEnc *e, XzbMfView &mf, uint32_t *back_res, uint32_t *len_res, uint32_t position)  // :802-858
{
	if (e->opts_end_index != e->opts_current_index) {
		*len_res = e->opts[e->opts_current_index].pos_prev - e->opts_current_index;
		*back_res = e->opts[e->opts_current_index].back_prev;
		e->opts_current_index = e->opts[e->opts_current_index].pos_prev;
		return;
	}
	if (mf.read_ahead == 0) {
		if (e->match_price_count >= (1 << 7)) xzb_fill_dist_prices(e);
		if (e->align_price_count >= XZB_ALIGN_SIZE) xzb_fill_align_prices(e);
	}
	uint32_t len_end = xzb_helper1(e, mf, back_res, len_res, position);
	if (len_end == 0xFFFFFFFFu) return;
	uint32_t reps[XZB_REPS];
	for (int i = 0; i < XZB_REPS; ++i) reps[i] = e->reps[i];
	uint32_t cur;
	for (cur = 1; cur < len_end; ++cur) {
		e->longest_match_length = xzb_mfv_find(mf, &e->matches_count, e->matches);
		if (e->longest_match_length >= mf.nice_len) break;
		len_end = xzb_helper2(e, reps, mf.buf + mf.read_pos - 1, len_end, position + cur, cur, mf.nice_len,
				xzb_min(xzb_mfv_avail(mf) + 1, XZB_OPTS - 1 - cur));
	}
	xzb_backward(e, len_res, back_res, cur);
}

// ------------------------------------------------------------------------------------
// lzma_lzma_encode (lzma/lzma_encoder.c:266-436) for one LZMA2 chunk, whole block resident
// ------------------------------------------------------------------------------------
XZB_HD_NOINLINE void xzb_lzma_encode_chunk(XzbEnc *e, XzbMfView &mf, uint32_t limit)
{
	if (!e->is_initialized) {  // encode_init :266-293
		if (mf.read_pos != mf.size) {
			xzb_mfv_skip(mf, 1);
			mf.read_ahead = 0;
			xzb_rc_bit(e->rc, &e->is_match[0][0], 0);
			xzb_rc_bittree(e->rc, e->literal + 0, 8, mf.buf[0]);
			++e->uncomp_size;
		}
		e->is_initialized = 1;
	}
	for (;;) {
		if (mf.read_pos - mf.read_ahead >= limit
				|| e->rc.out_pos + xzb_rc_pending(e->rc) >= XZB_LZMA2_CHUNK_MAX - XZB_LOOP_INPUT_MAX)
			break;  // :343-351
		if (mf.read_pos >= mf.size) {  // :354-360
			if (mf.read_ahead == 0) break;
		}
		uint32_t len, back;
		if (e->fast_mode) xzb_optimum_fast(e, mf, &back, &len);
		else xzb_optimum_normal(e, mf, &back, &len, (uint32_t)e->uncomp_size);
		xzb_encode_symbol(e, mf, back, len, (uint32_t)e->uncomp_size);
		e->uncomp_size += len;
	}
	xzb_rc_flush(e->rc);  // :427-437
}

// ------------------------------------------------------------------------------------
// lzma2_encode (lzma/lzma2_encoder.c:134-259, headers :53-131) over the whole block.
// Compressed bytes are range-coded straight into `out` behind a header slot whose size is
// known when the chunk starts (6 bytes with properties, 5 without).
// Returns XZB_OK, or XZB_BUF_ERROR when `out_cap` would be exceeded (the caller then takes
// the reference's "incompressible block" fallback, stream_encoder_mt.c:316-344).
// ------------------------------------------------------------------------------------
XZB_HD_NOINLINE int xzb_lzma2_encode_block(XzbEnc *e, XzbMfView &mf, uint8_t *out, uint32_t out_cap, uint32_t *out_pos_ptr)
{
	uint32_t out_pos = *out_pos_ptr;
	bool need_properties = true, need_state_reset = false, need_dictionary_reset = true;
	for (;;) {
		if (mf.size - mf.read_pos + mf.read_ahead == 0) {  // SEQ_INIT :146-161
			if (out_pos >= out_cap) return XZB_BUF_ERROR;
			out[out_pos++] = 0;
			break;
		}
		if (out_pos + XZB_LZMA2_HEADER_MAX + XZB_LZMA2_CHUNK_MAX > out_cap) return XZB_BUF_ERROR;
		if (need_state_reset) xzb_enc_reset(e);
		const uint32_t hdr = need_properties ? 6u : 5u;
		const uint32_t limit = mf.read_pos - mf.read_ahead + XZB_LZMA2_UNCOMPRESSED_MAX - XZB_MATCH_LEN_MAX;  // :163-181
		const uint32_t read_start = mf.read_pos - mf.read_ahead;
		e->rc.out = out + out_pos + hdr; e->rc.out_pos = 0;
		xzb_lzma_encode_chunk(e, mf, limit);
		const uint32_t compressed_size = e->rc.out_pos;
		uint32_t uncompressed_size = mf.read_pos - mf.read_ahead - read_start;
		if (compressed_size >= uncompressed_size) {
			// uncompressed chunk :202-214, header :107-131, payload via mf_read (lz_encoder.h:302-318)
			++e->n_chunks_raw;
			uncompressed_size += mf.read_ahead;
			mf.read_ahead = 0;
			out[out_pos++] = need_dictionary_reset ? 1 : 2;
			need_dictionary_reset = false;
			out[out_pos++] = (uint8_t)((uncompressed_size - 1) >> 8);
			out[out_pos++] = (uint8_t)((uncompressed_size - 1) & 0xFF);
			need_state_reset = true;
			const uint8_t *src = mf.buf + mf.read_pos - uncompressed_size;
			for (uint32_t i = 0; i < uncompressed_size; ++i) out[out_pos + i] = src[i];
			out_pos += uncompressed_size;
			continue;
		}
		++e->n_chunks_lzma;  // lzma2_header_lzma :53-104
		uint8_t *h = out + out_pos;
		uint32_t pos = 0;
		if (need_properties) h[pos] = need_dictionary_reset ? 0x80 + (3 << 5) : 0x80 + (2 << 5);
		else h[pos] = need_state_reset ? 0x80 + (1 << 5) : 0x80;
		uint32_t size = uncompressed_size - 1;
		h[pos++] += (uint8_t)(size >> 16);
		h[pos++] = (uint8_t)((size >> 8) & 0xFF);
		h[pos++] = (uint8_t)(size & 0xFF);
		size = compressed_size - 1;
		h[pos++] = (uint8_t)(size >> 8);
		h[pos++] = (uint8_t)(size & 0xFF);
		if (need_properties) h[pos++] = e->P.lclppb;
		need_properties = false; need_state_reset = false; need_dictionary_reset = false;
		out_pos += hdr + compressed_size;
	}
	*out_pos_ptr = out_pos;
	return XZB_OK;
}
