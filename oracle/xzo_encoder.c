/*
 * oracle/xzo_encoder.c -- CPU restatement of the reference's .xz/LZMA2 ENCODER path.
 *
 * TEST INFRASTRUCTURE ONLY (see oracle/xzo.h).  Sequential, whole-block-resident
 * restatement: the window never slides (SURVEY D5) and son[] has one slot per block
 * position instead of a cyclic buffer (SURVEY D8); everything else follows the
 * reference statement by statement.  Every function cites the reference lines
 * (relative to /root/reference/src/liblzma/) it restates.
 */
#include "xzo.h"
#include "xzo_tables.h"

#include <stdlib.h>
#include <string.h>

#define REPS 4
#define MATCH_LEN_MIN 2
#define MATCH_LEN_MAX 273
#define OPTS 4096
#define STATES 12
#define LIT_STATES 7
#define POS_STATES_MAX 16
#define LEN_LOW 8
#define LEN_MID 8
#define LEN_HIGH 256
#define LEN_SYMBOLS (LEN_LOW + LEN_MID + LEN_HIGH)
#define DIST_STATES 4
#define DIST_SLOTS 64
#define DIST_MODEL_START 4
#define DIST_MODEL_END 14
#define FULL_DISTANCES 128
#define ALIGN_BITS 4
#define ALIGN_SIZE 16
#define ALIGN_MASK 15
#define INFINITY_PRICE (1u << 30)
#define LZMA2_CHUNK_MAX (1u << 16)
#define LZMA2_UNCOMPRESSED_MAX (1u << 21)
#define LZMA2_HEADER_MAX 6
#define LOOP_INPUT_MAX (OPTS + 1)
#define BACK_LITERAL UINT32_MAX

typedef uint16_t prob_t;
typedef struct { uint32_t len, dist; } match_t;

/* ------------------------------------------------------------------ */
/* Symbol trace (debug aid for diffing parses)                         */
/* ------------------------------------------------------------------ */
static uint32_t *g_trace; static size_t g_trace_cap; static size_t *g_trace_count;
void xzo_set_trace(uint32_t *t, size_t cap, size_t *count) { g_trace = t; g_trace_cap = cap; g_trace_count = count; if (count) *count = 0; }

/* ------------------------------------------------------------------ */
/* Presets: lzma/lzma_encoder_presets.c:16-63                          */
/* ------------------------------------------------------------------ */
int xzo_lzma_preset(xzo_lzma_options *o, uint32_t preset)
{
	const uint32_t level = preset & 0x1F, flags = preset & ~0x1Fu;
	if (level > 9 || (flags & ~XZO_PRESET_EXTREME)) return 1;
	static const uint8_t dict_pow2[] = { 18, 20, 21, 22, 22, 23, 23, 24, 25, 26 };
	o->lc = 3; o->lp = 0; o->pb = 2;
	o->dict_size = 1u << dict_pow2[level];
	if (level <= 3) {
		static const uint8_t depths[] = { 4, 8, 24, 48 };
		o->mode = XZO_MODE_FAST;
		o->mf = level == 0 ? XZO_MF_HC3 : XZO_MF_HC4;
		o->nice_len = level <= 1 ? 128 : 273;
		o->depth = depths[level];
	} else {
		o->mode = XZO_MODE_NORMAL;
		o->mf = XZO_MF_BT4;
		o->nice_len = level == 4 ? 16 : level == 5 ? 32 : 64;
		o->depth = 0;
	}
	if (flags & XZO_PRESET_EXTREME) {
		o->mode = XZO_MODE_NORMAL;
		o->mf = XZO_MF_BT4;
		if (level == 3 || level == 5) { o->nice_len = 192; o->depth = 0; }
		else { o->nice_len = 273; o->depth = 512; }
	}
	return 0;
}

/* ------------------------------------------------------------------ */
/* Match finders: lz/lz_encoder.c:191-461, lz/lz_encoder_mf.c          */
/* ------------------------------------------------------------------ */
typedef struct {
	const uint8_t *buf;
	uint32_t size;          /* write_pos: the whole block is resident */
	uint32_t read_pos, read_ahead;
	uint32_t cyclic_size, hash_mask, depth, nice_len, mf, hash_bytes, is_bt;
	uint32_t *hash;         /* [h2:1024][h3:65536][main], value = position+1, 0 = EMPTY */
	uint32_t hash_count;
	uint32_t *son;          /* one slot (hc) / two slots (bt) per block position (D8) */
	xzo_counters *ctr;
} mf_t;

#define H2_SIZE 1024u
#define H3_SIZE 65536u

/* lz_encoder.c:191-368 (lz_encoder_prepare) + :371-461 (lz_encoder_init) */
static int mf_init(mf_t *mf, const uint8_t *buf, uint32_t size, const xzo_lzma_options *o, xzo_counters *ctr)
{
	memset(mf, 0, sizeof(*mf));
	mf->buf = buf; mf->size = size; mf->ctr = ctr;
	mf->mf = o->mf; mf->hash_bytes = o->mf & 0x0F; mf->is_bt = (o->mf & 0x10) != 0;
	/* lzma_encoder.c:486-502 set_lz_options: nice_len = max(hash_bytes, nice_len) */
	mf->nice_len = o->nice_len > mf->hash_bytes ? o->nice_len : mf->hash_bytes;
	mf->cyclic_size = o->dict_size + 1;
	uint32_t hs;
	if (mf->hash_bytes == 2) {
		hs = 0xFFFF;
	} else {
		hs = o->dict_size - 1;
		hs |= hs >> 1; hs |= hs >> 2; hs |= hs >> 4; hs |= hs >> 8;
		hs >>= 1; hs |= 0xFFFF;
		if (hs > (1u << 24)) { if (mf->hash_bytes == 3) hs = (1u << 24) - 1; else hs >>= 1; }
	}
	mf->hash_mask = hs;
	++hs;
	if (mf->hash_bytes > 2) hs += H2_SIZE;
	if (mf->hash_bytes > 3) hs += H3_SIZE;
	mf->hash_count = hs;
	mf->depth = o->depth;
	if (mf->depth == 0) mf->depth = mf->is_bt ? 16 + mf->nice_len / 2 : 4 + mf->nice_len / 4;
	mf->hash = calloc(hs, sizeof(uint32_t));
	mf->son = malloc(((size_t)size + 1) * (mf->is_bt ? 2 : 1) * sizeof(uint32_t));
	return mf->hash == NULL || mf->son == NULL;
}

static void mf_free(mf_t *mf) { free(mf->hash); free(mf->son); }

/* common/memcmplen.h:52-190: first index >= len where a and b differ, capped at limit */
static inline uint32_t memcmplen(const uint8_t *a, const uint8_t *b, uint32_t len, uint32_t limit)
{
	while (len < limit && a[len] == b[len]) ++len;
	return len;
}

static inline uint32_t mf_avail(const mf_t *mf) { return mf->size - mf->read_pos; }

/*
 * One match-finder step at read_pos: the find functions (lz_encoder_mf.c:303-334 hc3,
 * :365-413 hc4, :586-597 bt2, :619-649 bt3, :674-722 bt4) when m != NULL, the skip
 * functions (:337-360, :416-440, :600-614, :652-669, :725-743) when m == NULL.
 * Inner loops: hc_find_func :249-287, bt_find_func :449-512, bt_skip_func :515-568.
 * Positions are stored +1 so that 0 plays EMPTY_HASH_VALUE (:85); "delta >= cyclic_size"
 * (:266, :470) is evaluated on true distances, which equals the reference's test since
 * its offset is the same for both operands.
 */
static uint32_t mf_step(mf_t *mf, match_t *m)
{
	/* header() macro, :190-201 */
	uint32_t len_limit = mf_avail(mf);
	if (mf->nice_len <= len_limit) {
		len_limit = mf->nice_len;
	} else if (len_limit < mf->hash_bytes) {
		++mf->read_pos; /* move_pending(), :176-182: position is never inserted */
		return 0;
	}
	const uint8_t *cur = mf->buf + mf->read_pos;
	const uint32_t pos = mf->read_pos + 1; /* stored form */
	uint32_t count = 0;
	uint32_t len_best;
	uint32_t cur_match;
	int skip_tree = 0; /* len_best == len_limit after the head stage -> *_skip() (:327-330 etc.) */
	if (mf->ctr) mf->ctr->n_pos++;

	if (mf->hash_bytes == 2) {
		/* hash_2_calc, lz_encoder_hash.h:53-60 */
		const uint32_t hv = cur[0] | ((uint32_t)cur[1] << 8);
		cur_match = mf->hash[hv]; mf->hash[hv] = pos;
		len_best = 1;
	} else if (mf->hash_bytes == 3) {
		/* hash_3_calc, lz_encoder_hash.h:62-67 */
		const uint32_t temp = xzo_crc32_table[cur[0]] ^ cur[1];
		const uint32_t h2 = temp & (H2_SIZE - 1);
		const uint32_t hv = (temp ^ ((uint32_t)cur[2] << 8)) & mf->hash_mask;
		const uint32_t head2 = mf->hash[h2];
		cur_match = mf->hash[H2_SIZE + hv];
		mf->hash[h2] = pos; mf->hash[H2_SIZE + hv] = pos;
		len_best = 2;
		if (m != NULL) {
			const uint32_t delta2 = pos - head2;
			if (head2 != 0 && delta2 < mf->cyclic_size && *(cur - delta2) == *cur) {
				len_best = memcmplen(cur - delta2, cur, len_best, len_limit);
				m[0].len = len_best; m[0].dist = delta2 - 1; count = 1;
				if (len_best == len_limit) skip_tree = 1;
			}
		}
	} else {
		/* hash_4_calc, lz_encoder_hash.h:69-75 */
		const uint32_t temp = xzo_crc32_table[cur[0]] ^ cur[1];
		const uint32_t h2 = temp & (H2_SIZE - 1);
		const uint32_t h3 = (temp ^ ((uint32_t)cur[2] << 8)) & (H3_SIZE - 1);
		const uint32_t hv = (temp ^ ((uint32_t)cur[2] << 8) ^ (xzo_crc32_table[cur[3]] << 5)) & mf->hash_mask;
		const uint32_t head2 = mf->hash[h2], head3 = mf->hash[H2_SIZE + h3];
		cur_match = mf->hash[H2_SIZE + H3_SIZE + hv];
		mf->hash[h2] = pos; mf->hash[H2_SIZE + h3] = pos; mf->hash[H2_SIZE + H3_SIZE + hv] = pos;
		len_best = 1;
		if (m != NULL) {
			/* :372-410 / :681-719; an EMPTY head gives delta >= cyclic_size in the reference */
			uint32_t delta2 = head2 ? pos - head2 : UINT32_MAX;
			const uint32_t delta3 = head3 ? pos - head3 : UINT32_MAX;
			if (delta2 < mf->cyclic_size && *(cur - delta2) == *cur) {
				len_best = 2; m[0].len = 2; m[0].dist = delta2 - 1; count = 1;
			}
			if (delta2 != delta3 && delta3 < mf->cyclic_size && *(cur - delta3) == *cur) {
				len_best = 3; m[count++].dist = delta3 - 1; delta2 = delta3;
			}
			if (count != 0) {
				len_best = memcmplen(cur - delta2, cur, len_best, len_limit);
				m[count - 1].len = len_best;
				if (len_best == len_limit) skip_tree = 1;
			}
			if (len_best < 3) len_best = 3;
		}
	}

	const uint32_t p = mf->read_pos;
	uint32_t depth = mf->depth;

	if (!mf->is_bt) {
		/* hc_find_func :249-287 / hc_skip :294-298 */
		mf->son[p] = cur_match;
		if (m != NULL && !skip_tree) {
			match_t *out = m + count;
			for (;;) {
				const uint32_t delta = pos - cur_match;
				if (depth-- == 0 || cur_match == 0 || delta >= mf->cyclic_size) break;
				const uint8_t *pb = cur - delta;
				cur_match = mf->son[p - delta];
				if (mf->ctr) mf->ctr->n_nodes++;
				if (pb[len_best] == cur[len_best] && pb[0] == cur[0]) {
					const uint32_t len = memcmplen(pb, cur, 1, len_limit);
					if (mf->ctr) mf->ctr->n_cmp_bytes += len;
					if (len_best < len) {
						len_best = len; out->len = len; out->dist = delta - 1; ++out;
						if (len == len_limit) break;
					}
				}
			}
			count = (uint32_t)(out - m);
		}
	} else {
		/* bt_find_func :449-512 / bt_skip_func :515-568 */
		uint32_t *ptr0 = mf->son + ((size_t)p << 1) + 1;
		uint32_t *ptr1 = mf->son + ((size_t)p << 1);
		uint32_t len0 = 0, len1 = 0;
		const int record = (m != NULL && !skip_tree);
		match_t *out = m ? m + count : NULL;
		for (;;) {
			const uint32_t delta = pos - cur_match;
			if (depth-- == 0 || cur_match == 0 || delta >= mf->cyclic_size) {
				*ptr0 = 0; *ptr1 = 0;
				break;
			}
			uint32_t *pair = mf->son + ((size_t)(p - delta) << 1);
			const uint8_t *pb = cur - delta;
			uint32_t len = len0 < len1 ? len0 : len1;
			if (mf->ctr) mf->ctr->n_nodes++;
			if (pb[len] == cur[len]) {
				const uint32_t len_start = len;
				len = memcmplen(pb, cur, len + 1, len_limit);
				if (mf->ctr) mf->ctr->n_cmp_bytes += len - len_start;
				if (record) {
					if (len_best < len) {
						len_best = len; out->len = len; out->dist = delta - 1; ++out;
						if (len == len_limit) { *ptr1 = pair[0]; *ptr0 = pair[1]; break; }
					}
				} else if (len == len_limit) {
					*ptr1 = pair[0]; *ptr0 = pair[1]; break;
				}
			}
			if (pb[len] < cur[len]) {
				*ptr1 = cur_match; ptr1 = pair + 1; cur_match = *ptr1; len1 = len;
			} else {
				*ptr0 = cur_match; ptr0 = pair; cur_match = *ptr0; len0 = len;
			}
		}
		if (record) count = (uint32_t)(out - m);
	}
	++mf->read_pos; /* move_pos(), :148-159 (normalize never fires inside a block, D5) */
	return count;
}

/* lzma_mf_find, lz_encoder_mf.c:21-79 */
static uint32_t mf_find(mf_t *mf, uint32_t *count_ptr, match_t *matches)
{
	const uint32_t count = mf_step(mf, matches);
	uint32_t len_best = 0;
	if (count > 0) {
		len_best = matches[count - 1].len;
		if (len_best == mf->nice_len) {
			uint32_t limit = mf_avail(mf) + 1;
			if (limit > MATCH_LEN_MAX) limit = MATCH_LEN_MAX;
			const uint8_t *p1 = mf->buf + mf->read_pos - 1;
			const uint8_t *p2 = p1 - matches[count - 1].dist - 1;
			len_best = memcmplen(p1, p2, len_best, limit);
		}
		if (mf->ctr) mf->ctr->n_pairs += count;
	}
	*count_ptr = count;
	++mf->read_ahead;
	return len_best;
}

/* mf_skip, lz/lz_encoder.h:290-297 */
static void mf_skip(mf_t *mf, uint32_t amount)
{
	if (amount != 0) {
		for (uint32_t i = 0; i < amount; ++i) mf_step(mf, NULL);
		mf->read_ahead += amount;
	}
}

uint64_t xzo_mf_dump(const uint8_t *in, uint32_t n, const xzo_lzma_options *opt,
		uint32_t *counts, uint32_t *longest, uint64_t *offsets,
		uint32_t *pairs, uint64_t pairs_cap, xzo_counters *ctr)
{
	xzo_tables_init();
	mf_t mf;
	if (mf_init(&mf, in, n, opt, ctr)) return (uint64_t)-1;
	match_t m[MATCH_LEN_MAX + 1];
	uint64_t total = 0;
	for (uint32_t p = 0; p < n; ++p) {
		uint32_t c;
		const uint32_t lb = mf_find(&mf, &c, m);
		counts[p] = c; longest[p] = lb; offsets[p] = total;
		if (total + c > pairs_cap) { mf_free(&mf); return (uint64_t)-1; }
		for (uint32_t i = 0; i < c; ++i) { pairs[2 * (total + i)] = m[i].len; pairs[2 * (total + i) + 1] = m[i].dist; }
		total += c;
	}
	mf_free(&mf);
	return total;
}

/* ------------------------------------------------------------------ */
/* Range encoder: rangecoder/range_encoder.h                           */
/* The reference queues <= 53 symbols and drains them in rc_encode()    */
/* right after each LZMA symbol (lzma_encoder.c:404-419).  The only     */
/* reader of probabilities between queueing and draining is             */
/* length_update_prices() (see length_encode below); with that ordered  */
/* explicitly, encoding immediately is the same computation.            */
/* ------------------------------------------------------------------ */
typedef struct {
	uint64_t low, cache_size;
	uint32_t range;
	uint8_t cache;
	uint8_t *out; size_t out_pos; /* chunk buffer (lzma2_encoder.c:49) */
} rc_t;

/* rc_reset :62-72 */
static void rc_reset(rc_t *rc) { rc->low = 0; rc->cache_size = 1; rc->range = UINT32_MAX; rc->cache = 0; }

/* rc_shift_low :135-159 */
static void rc_shift_low(rc_t *rc)
{
	if ((uint32_t)rc->low < 0xFF000000u || (uint32_t)(rc->low >> 32) != 0) {
		do {
			rc->out[rc->out_pos++] = (uint8_t)(rc->cache + (uint8_t)(rc->low >> 32));
			rc->cache = 0xFF;
		} while (--rc->cache_size != 0);
		rc->cache = (rc->low >> 24) & 0xFF;
	}
	++rc->cache_size;
	rc->low = (rc->low & 0x00FFFFFF) << 8;
}

/* rc_bit :78-84 + rc_encode RC_BIT_0/1 :204-225 */
static inline void rc_bit(rc_t *rc, prob_t *prob, uint32_t bit)
{
	if (rc->range < (1u << 24)) { rc_shift_low(rc); rc->range <<= 8; }
	prob_t p = *prob;
	const uint32_t bound = (rc->range >> 11) * p;
	if (bit == 0) { rc->range = bound; p += (2048 - p) >> 5; }
	else { rc->low += bound; rc->range -= bound; p -= p >> 5; }
	*prob = p;
}

/* rc_bittree :87-98 */
static inline void rc_bittree(rc_t *rc, prob_t *probs, uint32_t bit_count, uint32_t symbol)
{
	uint32_t mi = 1;
	do {
		const uint32_t bit = (symbol >> --bit_count) & 1;
		rc_bit(rc, &probs[mi], bit);
		mi = (mi << 1) + bit;
	} while (bit_count != 0);
}

/* rc_bittree_reverse :101-113 */
static inline void rc_bittree_reverse(rc_t *rc, prob_t *probs, uint32_t bit_count, uint32_t symbol)
{
	uint32_t mi = 1;
	do {
		const uint32_t bit = symbol & 1; symbol >>= 1;
		rc_bit(rc, &probs[mi], bit);
		mi = (mi << 1) + bit;
	} while (--bit_count != 0);
}

/* rc_direct :116-124 + rc_encode RC_DIRECT_0/1 :227-234 */
static inline void rc_direct(rc_t *rc, uint32_t value, uint32_t bit_count)
{
	do {
		if (rc->range < (1u << 24)) { rc_shift_low(rc); rc->range <<= 8; }
		rc->range >>= 1;
		if ((value >> --bit_count) & 1) rc->low += rc->range;
	} while (bit_count != 0);
}

/* rc_flush :127-132 + rc_encode RC_FLUSH :236-249 (normalise first, :198-203) */
static void rc_flush(rc_t *rc)
{
	if (rc->range < (1u << 24)) { rc_shift_low(rc); rc->range <<= 8; }
	for (int i = 0; i < 5; ++i) rc_shift_low(rc);
	rc_reset(rc);
}

/* rc_pending :343-347 */
static inline uint64_t rc_pending(const rc_t *rc) { return rc->cache_size + 5 - 1; }

/* prices: rangecoder/price.h:28-90 */
static inline uint32_t pr_bit(prob_t p, uint32_t bit) { return xzo_rc_prices[(p ^ ((0u - bit) & 2047)) >> 4]; }
static inline uint32_t pr_bit0(prob_t p) { return xzo_rc_prices[p >> 4]; }
static inline uint32_t pr_bit1(prob_t p) { return xzo_rc_prices[(p ^ 2047) >> 4]; }
static inline uint32_t pr_bittree(const prob_t *probs, uint32_t levels, uint32_t symbol)
{
	uint32_t price = 0; symbol += 1u << levels;
	do { const uint32_t bit = symbol & 1; symbol >>= 1; price += pr_bit(probs[symbol], bit); } while (symbol != 1);
	return price;
}
static inline uint32_t pr_bittree_reverse(const prob_t *probs, uint32_t levels, uint32_t symbol)
{
	uint32_t price = 0, mi = 1;
	do { const uint32_t bit = symbol & 1; symbol >>= 1; price += pr_bit(probs[mi], bit); mi = (mi << 1) + bit; } while (--levels != 0);
	return price;
}
static inline uint32_t pr_direct(uint32_t bits) { return bits << 4; }

/* ------------------------------------------------------------------ */
/* LZMA encoder state: lzma/lzma_encoder_private.h:38-150              */
/* ------------------------------------------------------------------ */
typedef struct {
	prob_t choice, choice2;
	prob_t low[POS_STATES_MAX][LEN_LOW], mid[POS_STATES_MAX][LEN_MID], high[LEN_HIGH];
	uint32_t prices[POS_STATES_MAX][LEN_SYMBOLS];
	uint32_t table_size;
	uint32_t counters[POS_STATES_MAX];
} len_enc_t;

typedef struct {
	uint32_t state;
	uint8_t prev_1_is_literal, prev_2;
	uint32_t pos_prev_2, back_prev_2;
	uint32_t price, pos_prev, back_prev;
	uint32_t backs[REPS];
} optimal_t;

typedef struct {
	rc_t rc;
	uint64_t uncomp_size;
	uint32_t state;
	uint32_t reps[REPS];
	match_t matches[MATCH_LEN_MAX + 1];
	uint32_t matches_count, longest_match_length;
	int fast_mode, is_initialized;
	uint32_t pos_mask, lc, literal_mask;
	prob_t literal[16 * 0x300];
	prob_t is_match[STATES][POS_STATES_MAX];
	prob_t is_rep[STATES], is_rep0[STATES], is_rep1[STATES], is_rep2[STATES];
	prob_t is_rep0_long[STATES][POS_STATES_MAX];
	prob_t dist_slot[DIST_STATES][DIST_SLOTS];
	prob_t dist_special[FULL_DISTANCES - DIST_MODEL_END];
	prob_t dist_align[ALIGN_SIZE];
	len_enc_t match_len, rep_len;
	uint32_t dist_slot_prices[DIST_STATES][DIST_SLOTS];
	uint32_t dist_prices[DIST_STATES][FULL_DISTANCES];
	uint32_t dist_table_size, match_price_count;
	uint32_t align_prices[ALIGN_SIZE], align_price_count;
	uint32_t opts_end_index, opts_current_index;
	optimal_t opts[OPTS];
	xzo_lzma_options opt;
	xzo_counters *ctr;
} enc_t;

/* state machine: lzma/lzma_common.h:55-114 */
#define st_is_literal(s) ((s) < LIT_STATES)
static inline uint32_t st_literal(uint32_t s) { return s <= 3 ? 0 : (s <= 9 ? s - 3 : s - 6); }
static inline uint32_t st_match(uint32_t s) { return s < LIT_STATES ? 7 : 10; }
static inline uint32_t st_long_rep(uint32_t s) { return s < LIT_STATES ? 8 : 11; }
static inline uint32_t st_short_rep(uint32_t s) { return s < LIT_STATES ? 9 : 11; }
/* get_dist_state, lzma_common.h:185-188 */
static inline uint32_t dist_state_of(uint32_t len) { return len < DIST_STATES + MATCH_LEN_MIN ? len - MATCH_LEN_MIN : DIST_STATES - 1; }
/* literal_subcoder, lzma_common.h:141-143 */
static inline prob_t *lit_subcoder(enc_t *e, uint32_t pos, uint32_t prev_byte)
{
	return e->literal + 3u * ((((pos << 8) + prev_byte) & e->literal_mask) << e->lc);
}
/* get_dist_slot, lzma/fastpos.h:77-136 (table and bsr forms are the same function) */
static inline uint32_t dist_slot_of(uint32_t dist)
{
	if (dist <= 4) return dist;
	const uint32_t i = 31 - (uint32_t)__builtin_clz(dist);
	return (i + i) + ((dist >> (i - 1)) & 1);
}

/* length_update_prices, lzma/lzma_encoder.c:76-102 */
static void length_update_prices(len_enc_t *lc, uint32_t pos_state)
{
	const uint32_t table_size = lc->table_size;
	lc->counters[pos_state] = table_size;
	const uint32_t a0 = pr_bit0(lc->choice), a1 = pr_bit1(lc->choice);
	const uint32_t b0 = a1 + pr_bit0(lc->choice2), b1 = a1 + pr_bit1(lc->choice2);
	uint32_t *prices = lc->prices[pos_state];
	uint32_t i;
	for (i = 0; i < table_size && i < LEN_LOW; ++i) prices[i] = a0 + pr_bittree(lc->low[pos_state], 3, i);
	for (; i < table_size && i < LEN_LOW + LEN_MID; ++i) prices[i] = b0 + pr_bittree(lc->mid[pos_state], 3, i - LEN_LOW);
	for (; i < table_size; ++i) prices[i] = b1 + pr_bittree(lc->high, 8, i - LEN_LOW - LEN_MID);
}

/* length, lzma_encoder.c:105-134.  NOTE on ordering: the reference only QUEUES the bits
 * here (rc_bit, range_encoder.h:78-84) and applies them to the probabilities later in
 * rc_encode(); so when the counter reaches zero, length_update_prices() still sees the
 * probabilities from BEFORE this length's own bits.  We encode immediately, hence the
 * price refresh has to run first. */
static void length_encode(enc_t *e, len_enc_t *lc, uint32_t pos_state, uint32_t len)
{
	rc_t *rc = &e->rc;
	if (!e->fast_mode)
		if (--lc->counters[pos_state] == 0)
			length_update_prices(lc, pos_state);
	len -= MATCH_LEN_MIN;
	if (len < LEN_LOW) {
		rc_bit(rc, &lc->choice, 0);
		rc_bittree(rc, lc->low[pos_state], 3, len);
	} else {
		rc_bit(rc, &lc->choice, 1);
		len -= LEN_LOW;
		if (len < LEN_MID) {
			rc_bit(rc, &lc->choice2, 0);
			rc_bittree(rc, lc->mid[pos_state], 3, len);
		} else {
			rc_bit(rc, &lc->choice2, 1);
			len -= LEN_MID;
			rc_bittree(rc, lc->high, 8, len);
		}
	}
}

/* length_encoder_reset, lzma_encoder.c:505-525 */
static void len_reset(len_enc_t *lc, uint32_t num_pos_states, int fast_mode)
{
	lc->choice = 1024; lc->choice2 = 1024;
	for (uint32_t ps = 0; ps < num_pos_states; ++ps) {
		for (int i = 0; i < LEN_LOW; ++i) lc->low[ps][i] = 1024;
		for (int i = 0; i < LEN_MID; ++i) lc->mid[ps][i] = 1024;
	}
	for (int i = 0; i < LEN_HIGH; ++i) lc->high[i] = 1024;
	if (!fast_mode)
		for (uint32_t ps = 0; ps < num_pos_states; ++ps) length_update_prices(lc, ps);
}

/* lzma_lzma_encoder_reset, lzma_encoder.c:528-598 */
static void enc_reset(enc_t *e)
{
	const xzo_lzma_options *o = &e->opt;
	e->pos_mask = (1u << o->pb) - 1;
	e->lc = o->lc;
	e->literal_mask = (0x100u << o->lp) - (0x100u >> o->lc);
	rc_reset(&e->rc);
	e->state = 0;
	for (int i = 0; i < REPS; ++i) e->reps[i] = 0;
	const size_t coders = (size_t)0x300 << (o->lc + o->lp);
	for (size_t i = 0; i < coders; ++i) e->literal[i] = 1024;
	for (int i = 0; i < STATES; ++i) {
		for (uint32_t j = 0; j <= e->pos_mask; ++j) { e->is_match[i][j] = 1024; e->is_rep0_long[i][j] = 1024; }
		e->is_rep[i] = e->is_rep0[i] = e->is_rep1[i] = e->is_rep2[i] = 1024;
	}
	for (int i = 0; i < FULL_DISTANCES - DIST_MODEL_END; ++i) e->dist_special[i] = 1024;
	for (int i = 0; i < DIST_STATES; ++i) for (int j = 0; j < DIST_SLOTS; ++j) e->dist_slot[i][j] = 1024;
	for (int i = 0; i < ALIGN_SIZE; ++i) e->dist_align[i] = 1024;
	len_reset(&e->match_len, 1u << o->pb, e->fast_mode);
	len_reset(&e->rep_len, 1u << o->pb, e->fast_mode);
	e->match_price_count = UINT32_MAX / 2;
	e->align_price_count = UINT32_MAX / 2;
	e->opts_end_index = 0; e->opts_current_index = 0;
}

/* lzma_lzma_encoder_create, lzma_encoder.c:601-707 */
static int enc_create(enc_t *e, const xzo_lzma_options *o, xzo_counters *ctr)
{
	e->opt = *o; e->ctr = ctr;
	if (o->lc > 4 || o->lp > 4 || o->lc + o->lp > 4 || o->pb > 4) return XZO_OPTIONS_ERROR;
	if (o->nice_len < MATCH_LEN_MIN || o->nice_len > MATCH_LEN_MAX) return XZO_OPTIONS_ERROR;
	const uint32_t hash_bytes = o->mf & 0x0F;
	const uint32_t nice_len = o->nice_len > hash_bytes ? o->nice_len : hash_bytes;
	if (o->mode == XZO_MODE_FAST) {
		e->fast_mode = 1;
	} else if (o->mode == XZO_MODE_NORMAL) {
		e->fast_mode = 0;
		if (o->dict_size > (1u << 30) + (1u << 29)) return XZO_OPTIONS_ERROR;
		uint32_t log_size = 0;
		while ((1u << log_size) < o->dict_size) ++log_size;
		e->dist_table_size = log_size * 2;
		e->match_len.table_size = nice_len + 1 - MATCH_LEN_MIN;
		e->rep_len.table_size = nice_len + 1 - MATCH_LEN_MIN;
	} else {
		return XZO_OPTIONS_ERROR;
	}
	e->is_initialized = 0;
	e->uncomp_size = 0;
	enc_reset(e);
	return XZO_OK;
}

/* literal_matched :22-43, literal :46-69 */
static void literal_encode(enc_t *e, const mf_t *mf, uint32_t position)
{
	const uint8_t cur_byte = mf->buf[mf->read_pos - mf->read_ahead];
	prob_t *sub = lit_subcoder(e, position, mf->buf[mf->read_pos - mf->read_ahead - 1]);
	if (st_is_literal(e->state)) {
		e->state = e->state <= 3 ? 0 : e->state - 3; /* update_literal_normal */
		rc_bittree(&e->rc, sub, 8, cur_byte);
	} else {
		e->state = e->state <= 9 ? e->state - 3 : e->state - 6; /* update_literal_matched */
		uint32_t match_byte = mf->buf[mf->read_pos - e->reps[0] - 1 - mf->read_ahead];
		uint32_t offset = 0x100, symbol = cur_byte + (1u << 8);
		do {
			match_byte <<= 1;
			const uint32_t match_bit = match_byte & offset;
			const uint32_t idx = offset + match_bit + (symbol >> 8);
			const uint32_t bit = (symbol >> 7) & 1;
			rc_bit(&e->rc, &sub[idx], bit);
			symbol <<= 1;
			offset &= ~(match_byte ^ symbol);
		} while (symbol < (1u << 16));
	}
}

/* match, lzma_encoder.c:141-181 */
static void match_encode(enc_t *e, uint32_t pos_state, uint32_t distance, uint32_t len)
{
	e->state = st_match(e->state);
	length_encode(e, &e->match_len, pos_state, len);
	const uint32_t slot = dist_slot_of(distance);
	rc_bittree(&e->rc, e->dist_slot[dist_state_of(len)], 6, slot);
	if (slot >= DIST_MODEL_START) {
		const uint32_t footer_bits = (slot >> 1) - 1;
		const uint32_t base = (2 | (slot & 1)) << footer_bits;
		const uint32_t reduced = distance - base;
		if (slot < DIST_MODEL_END) {
			rc_bittree_reverse(&e->rc, e->dist_special + base - slot - 1, footer_bits, reduced);
		} else {
			rc_direct(&e->rc, reduced >> ALIGN_BITS, footer_bits - ALIGN_BITS);
			rc_bittree_reverse(&e->rc, e->dist_align, ALIGN_BITS, reduced & ALIGN_MASK);
			++e->align_price_count;
		}
	}
	e->reps[3] = e->reps[2]; e->reps[2] = e->reps[1]; e->reps[1] = e->reps[0]; e->reps[0] = distance;
	++e->match_price_count;
}

/* rep_match, lzma_encoder.c:188-225 */
static void rep_match_encode(enc_t *e, uint32_t pos_state, uint32_t rep, uint32_t len)
{
	rc_t *rc = &e->rc;
	if (rep == 0) {
		rc_bit(rc, &e->is_rep0[e->state], 0);
		rc_bit(rc, &e->is_rep0_long[e->state][pos_state], len != 1);
	} else {
		const uint32_t distance = e->reps[rep];
		rc_bit(rc, &e->is_rep0[e->state], 1);
		if (rep == 1) {
			rc_bit(rc, &e->is_rep1[e->state], 0);
		} else {
			rc_bit(rc, &e->is_rep1[e->state], 1);
			rc_bit(rc, &e->is_rep2[e->state], rep - 2);
			if (rep == 3) e->reps[3] = e->reps[2];
			e->reps[2] = e->reps[1];
		}
		e->reps[1] = e->reps[0];
		e->reps[0] = distance;
	}
	if (len == 1) {
		e->state = st_short_rep(e->state);
	} else {
		length_encode(e, &e->rep_len, pos_state, len);
		e->state = st_long_rep(e->state);
	}
}

/* encode_symbol, lzma_encoder.c:232-263 */
static void encode_symbol(enc_t *e, mf_t *mf, uint32_t back, uint32_t len, uint32_t position)
{
	const uint32_t pos_state = position & e->pos_mask;
	if (g_trace && g_trace_count && *g_trace_count < g_trace_cap) {
		uint32_t *t = g_trace + 3 * (*g_trace_count)++;
		t[0] = mf->read_pos - mf->read_ahead; t[1] = back; t[2] = len;
	}
	if (e->ctr) e->ctr->n_symbols++;
	if (back == BACK_LITERAL) {
		rc_bit(&e->rc, &e->is_match[e->state][pos_state], 0);
		literal_encode(e, mf, position);
	} else {
		rc_bit(&e->rc, &e->is_match[e->state][pos_state], 1);
		if (back < REPS) {
			rc_bit(&e->rc, &e->is_rep[e->state], 1);
			rep_match_encode(e, pos_state, back, len);
		} else {
			rc_bit(&e->rc, &e->is_rep[e->state], 0);
			match_encode(e, pos_state, back - REPS, len);
		}
	}
	mf->read_ahead -= len;
}

/* ------------------------------------------------------------------ */
/* lzma_lzma_optimum_fast: lzma/lzma_encoder_optimum_fast.c:19-169     */
/* ------------------------------------------------------------------ */
#define change_pair(small_dist, big_dist) (((big_dist) >> 7) > (small_dist))
static inline int ne16(const uint8_t *a, const uint8_t *b) { return a[0] != b[0] || a[1] != b[1]; }

static void optimum_fast(enc_t *e, mf_t *mf, uint32_t *back_res, uint32_t *len_res)
{
	const uint32_t nice_len = mf->nice_len;
	uint32_t len_main, matches_count;
	if (mf->read_ahead == 0) {
		len_main = mf_find(mf, &matches_count, e->matches);
	} else {
		len_main = e->longest_match_length;
		matches_count = e->matches_count;
	}
	const uint8_t *buf = mf->buf + mf->read_pos - 1;
	const uint32_t buf_avail = mf_avail(mf) + 1 < MATCH_LEN_MAX ? mf_avail(mf) + 1 : MATCH_LEN_MAX;
	if (buf_avail < 2) { *back_res = BACK_LITERAL; *len_res = 1; return; }

	uint32_t rep_len = 0, rep_index = 0;
	for (uint32_t i = 0; i < REPS; ++i) {
		const uint8_t *bb = buf - e->reps[i] - 1;
		if (ne16(buf, bb)) continue;
		const uint32_t len = memcmplen(buf, bb, 2, buf_avail);
		if (len >= nice_len) { *back_res = i; *len_res = len; mf_skip(mf, len - 1); return; }
		if (len > rep_len) { rep_index = i; rep_len = len; }
	}
	if (len_main >= nice_len) {
		*back_res = e->matches[matches_count - 1].dist + REPS; *len_res = len_main;
		mf_skip(mf, len_main - 1); return;
	}
	uint32_t back_main = 0;
	if (len_main >= 2) {
		back_main = e->matches[matches_count - 1].dist;
		while (matches_count > 1 && len_main == e->matches[matches_count - 2].len + 1) {
			if (!change_pair(e->matches[matches_count - 2].dist, back_main)) break;
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
			*back_res = rep_index; *len_res = rep_len; mf_skip(mf, rep_len - 1); return;
		}
	}
	if (len_main < 2 || buf_avail <= 2) { *back_res = BACK_LITERAL; *len_res = 1; return; }

	e->longest_match_length = mf_find(mf, &e->matches_count, e->matches);
	if (e->longest_match_length >= 2) {
		const uint32_t new_dist = e->matches[e->matches_count - 1].dist;
		if ((e->longest_match_length >= len_main && new_dist < back_main)
				|| (e->longest_match_length == len_main + 1 && !change_pair(back_main, new_dist))
				|| (e->longest_match_length > len_main + 1)
				|| (e->longest_match_length + 1 >= len_main && len_main >= 3 && change_pair(new_dist, back_main))) {
			*back_res = BACK_LITERAL; *len_res = 1; return;
		}
	}
	++buf;
	const uint32_t limit = len_main - 1 > 2 ? len_main - 1 : 2;
	for (uint32_t i = 0; i < REPS; ++i) {
		if (memcmp(buf, buf - e->reps[i] - 1, limit) == 0) { *back_res = BACK_LITERAL; *len_res = 1; return; }
	}
	*back_res = back_main + REPS; *len_res = len_main;
	mf_skip(mf, len_main - 2);
}

/* ------------------------------------------------------------------ */
/* lzma_lzma_optimum_normal: lzma/lzma_encoder_optimum_normal.c        */
/* ------------------------------------------------------------------ */
/* get_literal_price :20-53 */
static uint32_t literal_price(enc_t *e, uint32_t pos, uint32_t prev_byte, int match_mode, uint32_t match_byte, uint32_t symbol)
{
	const prob_t *sub = lit_subcoder(e, pos, prev_byte);
	uint32_t price = 0;
	if (!match_mode) {
		price = pr_bittree(sub, 8, symbol);
	} else {
		uint32_t offset = 0x100; symbol += 1u << 8;
		do {
			match_byte <<= 1;
			const uint32_t match_bit = match_byte & offset;
			const uint32_t idx = offset + match_bit + (symbol >> 8);
			const uint32_t bit = (symbol >> 7) & 1;
			price += pr_bit(sub[idx], bit);
			symbol <<= 1;
			offset &= ~(match_byte ^ symbol);
		} while (symbol < (1u << 16));
	}
	return price;
}
/* get_len_price :56-63 */
static inline uint32_t len_price(const len_enc_t *l, uint32_t len, uint32_t ps) { return l->prices[ps][len - MATCH_LEN_MIN]; }
/* get_short_rep_price :66-72 */
static inline uint32_t short_rep_price(const enc_t *e, uint32_t st, uint32_t ps) { return pr_bit0(e->is_rep0[st]) + pr_bit0(e->is_rep0_long[st][ps]); }
/* get_pure_rep_price :75-97 */
static uint32_t pure_rep_price(const enc_t *e, uint32_t rep, uint32_t st, uint32_t ps)
{
	uint32_t price;
	if (rep == 0) {
		price = pr_bit0(e->is_rep0[st]) + pr_bit1(e->is_rep0_long[st][ps]);
	} else {
		price = pr_bit1(e->is_rep0[st]);
		if (rep == 1) price += pr_bit0(e->is_rep1[st]);
		else { price += pr_bit1(e->is_rep1[st]); price += pr_bit(e->is_rep2[st], rep - 2); }
	}
	return price;
}
/* get_rep_price :100-107 */
static inline uint32_t rep_price(const enc_t *e, uint32_t rep, uint32_t len, uint32_t st, uint32_t ps) { return len_price(&e->rep_len, len, ps) + pure_rep_price(e, rep, st, ps); }
/* get_dist_len_price :110-128 */
static uint32_t dist_len_price(const enc_t *e, uint32_t dist, uint32_t len, uint32_t ps)
{
	const uint32_t ds = dist_state_of(len);
	uint32_t price;
	if (dist < FULL_DISTANCES) price = e->dist_prices[ds][dist];
	else price = e->dist_slot_prices[ds][dist_slot_of(dist)] + e->align_prices[dist & ALIGN_MASK];
	return price + len_price(&e->match_len, len, ps);
}
/* fill_dist_prices :131-183 */
static void fill_dist_prices(enc_t *e)
{
	for (uint32_t ds = 0; ds < DIST_STATES; ++ds) {
		uint32_t *sp = e->dist_slot_prices[ds];
		for (uint32_t s = 0; s < e->dist_table_size; ++s) sp[s] = pr_bittree(e->dist_slot[ds], 6, s);
		for (uint32_t s = DIST_MODEL_END; s < e->dist_table_size; ++s) sp[s] += pr_direct(((s >> 1) - 1) - ALIGN_BITS);
		for (uint32_t i = 0; i < DIST_MODEL_START; ++i) e->dist_prices[ds][i] = sp[i];
	}
	for (uint32_t i = DIST_MODEL_START; i < FULL_DISTANCES; ++i) {
		const uint32_t slot = dist_slot_of(i);
		const uint32_t footer_bits = (slot >> 1) - 1;
		const uint32_t base = (2 | (slot & 1)) << footer_bits;
		const uint32_t price = pr_bittree_reverse(e->dist_special + base - slot - 1, footer_bits, i - base);
		for (uint32_t ds = 0; ds < DIST_STATES; ++ds) e->dist_prices[ds][i] = price + e->dist_slot_prices[ds][slot];
	}
	e->match_price_count = 0;
}
/* fill_align_prices :186-195 */
static void fill_align_prices(enc_t *e)
{
	for (uint32_t i = 0; i < ALIGN_SIZE; ++i) e->align_prices[i] = pr_bittree_reverse(e->dist_align, ALIGN_BITS, i);
	e->align_price_count = 0;
}

/* make_literal :202-208, make_short_rep :210-215 */
static inline void make_literal(optimal_t *o) { o->back_prev = BACK_LITERAL; o->prev_1_is_literal = 0; }
static inline void make_short_rep(optimal_t *o) { o->back_prev = 0; o->prev_1_is_literal = 0; }

/* backward :222-263 */
static void backward(enc_t *e, uint32_t *len_res, uint32_t *back_res, uint32_t cur)
{
	optimal_t *opts = e->opts;
	e->opts_end_index = cur;
	uint32_t pos_mem = opts[cur].pos_prev;
	uint32_t back_mem = opts[cur].back_prev;
	do {
		if (opts[cur].prev_1_is_literal) {
			make_literal(&opts[pos_mem]);
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

/* helper1 :270-439 */
static uint32_t helper1(enc_t *e, mf_t *mf, uint32_t *back_res, uint32_t *len_res, uint32_t position)
{
	optimal_t *opts = e->opts;
	const uint32_t nice_len = mf->nice_len;
	uint32_t len_main, matches_count;
	if (mf->read_ahead == 0) {
		len_main = mf_find(mf, &matches_count, e->matches);
	} else {
		len_main = e->longest_match_length;
		matches_count = e->matches_count;
	}
	const uint32_t buf_avail = mf_avail(mf) + 1 < MATCH_LEN_MAX ? mf_avail(mf) + 1 : MATCH_LEN_MAX;
	if (buf_avail < 2) { *back_res = BACK_LITERAL; *len_res = 1; return UINT32_MAX; }
	const uint8_t *buf = mf->buf + mf->read_pos - 1;

	uint32_t rep_lens[REPS];
	uint32_t rep_max_index = 0;
	for (uint32_t i = 0; i < REPS; ++i) {
		const uint8_t *bb = buf - e->reps[i] - 1;
		if (ne16(buf, bb)) { rep_lens[i] = 0; continue; }
		rep_lens[i] = memcmplen(buf, bb, 2, buf_avail);
		if (rep_lens[i] > rep_lens[rep_max_index]) rep_max_index = i;
	}
	if (rep_lens[rep_max_index] >= nice_len) {
		*back_res = rep_max_index; *len_res = rep_lens[rep_max_index];
		mf_skip(mf, *len_res - 1); return UINT32_MAX;
	}
	if (len_main >= nice_len) {
		*back_res = e->matches[matches_count - 1].dist + REPS; *len_res = len_main;
		mf_skip(mf, len_main - 1); return UINT32_MAX;
	}
	const uint8_t current_byte = *buf;
	const uint8_t match_byte = *(buf - e->reps[0] - 1);
	if (len_main < 2 && current_byte != match_byte && rep_lens[rep_max_index] < 2) {
		*back_res = BACK_LITERAL; *len_res = 1; return UINT32_MAX;
	}
	opts[0].state = e->state;
	const uint32_t pos_state = position & e->pos_mask;
	opts[1].price = pr_bit0(e->is_match[e->state][pos_state])
			+ literal_price(e, position, buf[-1], !st_is_literal(e->state), match_byte, current_byte);
	make_literal(&opts[1]);
	const uint32_t match_price = pr_bit1(e->is_match[e->state][pos_state]);
	const uint32_t rep_match_price = match_price + pr_bit1(e->is_rep[e->state]);
	if (match_byte == current_byte) {
		const uint32_t srp = rep_match_price + short_rep_price(e, e->state, pos_state);
		if (srp < opts[1].price) { opts[1].price = srp; make_short_rep(&opts[1]); }
	}
	const uint32_t len_end = len_main > rep_lens[rep_max_index] ? len_main : rep_lens[rep_max_index];
	if (len_end < 2) { *back_res = opts[1].back_prev; *len_res = 1; return UINT32_MAX; }
	opts[1].pos_prev = 0;
	for (uint32_t i = 0; i < REPS; ++i) opts[0].backs[i] = e->reps[i];
	uint32_t len = len_end;
	do { opts[len].price = INFINITY_PRICE; } while (--len >= 2);

	for (uint32_t i = 0; i < REPS; ++i) {
		uint32_t rep_len = rep_lens[i];
		if (rep_len < 2) continue;
		const uint32_t price = rep_match_price + pure_rep_price(e, i, e->state, pos_state);
		do {
			const uint32_t p = price + len_price(&e->rep_len, rep_len, pos_state);
			if (p < opts[rep_len].price) {
				opts[rep_len].price = p; opts[rep_len].pos_prev = 0;
				opts[rep_len].back_prev = i; opts[rep_len].prev_1_is_literal = 0;
			}
		} while (--rep_len >= 2);
	}
	const uint32_t normal_match_price = match_price + pr_bit0(e->is_rep[e->state]);
	len = rep_lens[0] >= 2 ? rep_lens[0] + 1 : 2;
	if (len <= len_main) {
		uint32_t i = 0;
		while (len > e->matches[i].len) ++i;
		for (;; ++len) {
			const uint32_t dist = e->matches[i].dist;
			const uint32_t p = normal_match_price + dist_len_price(e, dist, len, pos_state);
			if (p < opts[len].price) {
				opts[len].price = p; opts[len].pos_prev = 0;
				opts[len].back_prev = dist + REPS; opts[len].prev_1_is_literal = 0;
			}
			if (len == e->matches[i].len)
				if (++i == matches_count) break;
		}
	}
	return len_end;
}

/* helper2 :442-799 */
static uint32_t helper2(enc_t *e, uint32_t *reps, const uint8_t *buf, uint32_t len_end,
		uint32_t position, const uint32_t cur, const uint32_t nice_len, const uint32_t buf_avail_full)
{
	optimal_t *opts = e->opts;
	uint32_t matches_count = e->matches_count;
	uint32_t new_len = e->longest_match_length;
	uint32_t pos_prev = opts[cur].pos_prev;
	uint32_t state;

	if (opts[cur].prev_1_is_literal) {
		--pos_prev;
		if (opts[cur].prev_2) {
			state = opts[opts[cur].pos_prev_2].state;
			if (opts[cur].back_prev_2 < REPS) state = st_long_rep(state);
			else state = st_match(state);
		} else {
			state = opts[pos_prev].state;
		}
		state = st_literal(state);
	} else {
		state = opts[pos_prev].state;
	}

	if (pos_prev == cur - 1) {
		if (opts[cur].back_prev == 0) state = st_short_rep(state);
		else state = st_literal(state);
	} else {
		uint32_t pos;
		if (opts[cur].prev_1_is_literal && opts[cur].prev_2) {
			pos_prev = opts[cur].pos_prev_2;
			pos = opts[cur].back_prev_2;
			state = st_long_rep(state);
		} else {
			pos = opts[cur].back_prev;
			if (pos < REPS) state = st_long_rep(state);
			else state = st_match(state);
		}
		if (pos < REPS) {
			reps[0] = opts[pos_prev].backs[pos];
			uint32_t i;
			for (i = 1; i <= pos; ++i) reps[i] = opts[pos_prev].backs[i - 1];
			for (; i < REPS; ++i) reps[i] = opts[pos_prev].backs[i];
		} else {
			reps[0] = pos - REPS;
			for (uint32_t i = 1; i < REPS; ++i) reps[i] = opts[pos_prev].backs[i - 1];
		}
	}
	opts[cur].state = state;
	for (uint32_t i = 0; i < REPS; ++i) opts[cur].backs[i] = reps[i];

	const uint32_t cur_price = opts[cur].price;
	const uint8_t current_byte = *buf;
	const uint8_t match_byte = *(buf - reps[0] - 1);
	const uint32_t pos_state = position & e->pos_mask;
	const uint32_t cur_and_1_price = cur_price + pr_bit0(e->is_match[state][pos_state])
			+ literal_price(e, position, buf[-1], !st_is_literal(state), match_byte, current_byte);
	int next_is_literal = 0;
	if (cur_and_1_price < opts[cur + 1].price) {
		opts[cur + 1].price = cur_and_1_price;
		opts[cur + 1].pos_prev = cur;
		make_literal(&opts[cur + 1]);
		next_is_literal = 1;
	}
	const uint32_t match_price = cur_price + pr_bit1(e->is_match[state][pos_state]);
	const uint32_t rep_match_price = match_price + pr_bit1(e->is_rep[state]);
	if (match_byte == current_byte && !(opts[cur + 1].pos_prev < cur && opts[cur + 1].back_prev == 0)) {
		const uint32_t srp = rep_match_price + short_rep_price(e, state, pos_state);
		if (srp <= opts[cur + 1].price) {
			opts[cur + 1].price = srp;
			opts[cur + 1].pos_prev = cur;
			make_short_rep(&opts[cur + 1]);
			next_is_literal = 1;
		}
	}
	if (buf_avail_full < 2) return len_end;
	const uint32_t buf_avail = buf_avail_full < nice_len ? buf_avail_full : nice_len;

	if (!next_is_literal && match_byte != current_byte) {
		/* literal + rep0, :562-597 */
		const uint8_t *bb = buf - reps[0] - 1;
		const uint32_t limit = buf_avail_full < nice_len + 1 ? buf_avail_full : nice_len + 1;
		const uint32_t len_test = memcmplen(buf, bb, 1, limit) - 1;
		if (len_test >= 2) {
			const uint32_t state_2 = st_literal(state);
			const uint32_t psn = (position + 1) & e->pos_mask;
			const uint32_t nrmp = cur_and_1_price + pr_bit1(e->is_match[state_2][psn]) + pr_bit1(e->is_rep[state_2]);
			const uint32_t offset = cur + 1 + len_test;
			while (len_end < offset) opts[++len_end].price = INFINITY_PRICE;
			const uint32_t p = nrmp + rep_price(e, 0, len_test, state_2, psn);
			if (p < opts[offset].price) {
				opts[offset].price = p; opts[offset].pos_prev = cur + 1; opts[offset].back_prev = 0;
				opts[offset].prev_1_is_literal = 1; opts[offset].prev_2 = 0;
			}
		}
	}

	uint32_t start_len = 2;
	for (uint32_t rep_index = 0; rep_index < REPS; ++rep_index) {
		const uint8_t *bb = buf - reps[rep_index] - 1;
		if (ne16(buf, bb)) continue;
		uint32_t len_test = memcmplen(buf, bb, 2, buf_avail);
		while (len_end < cur + len_test) opts[++len_end].price = INFINITY_PRICE;
		const uint32_t len_test_temp = len_test;
		const uint32_t price = rep_match_price + pure_rep_price(e, rep_index, state, pos_state);
		do {
			const uint32_t p = price + len_price(&e->rep_len, len_test, pos_state);
			if (p < opts[cur + len_test].price) {
				opts[cur + len_test].price = p; opts[cur + len_test].pos_prev = cur;
				opts[cur + len_test].back_prev = rep_index; opts[cur + len_test].prev_1_is_literal = 0;
			}
		} while (--len_test >= 2);
		len_test = len_test_temp;
		if (rep_index == 0) start_len = len_test + 1;

		uint32_t len_test_2 = len_test + 1;
		const uint32_t limit = buf_avail_full < len_test_2 + nice_len ? buf_avail_full : len_test_2 + nice_len;
		if (len_test_2 < limit) len_test_2 = memcmplen(buf, bb, len_test_2, limit);
		len_test_2 -= len_test + 1;
		if (len_test_2 >= 2) {
			uint32_t state_2 = st_long_rep(state);
			uint32_t psn = (position + len_test) & e->pos_mask;
			const uint32_t calp = price + len_price(&e->rep_len, len_test, pos_state)
					+ pr_bit0(e->is_match[state_2][psn])
					+ literal_price(e, position + len_test, buf[len_test - 1], 1, bb[len_test], buf[len_test]);
			state_2 = st_literal(state_2);
			psn = (position + len_test + 1) & e->pos_mask;
			const uint32_t nrmp = calp + pr_bit1(e->is_match[state_2][psn]) + pr_bit1(e->is_rep[state_2]);
			const uint32_t offset = cur + len_test + 1 + len_test_2;
			while (len_end < offset) opts[++len_end].price = INFINITY_PRICE;
			const uint32_t p = nrmp + rep_price(e, 0, len_test_2, state_2, psn);
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
		const uint32_t normal_match_price = match_price + pr_bit0(e->is_rep[state]);
		while (len_end < cur + new_len) opts[++len_end].price = INFINITY_PRICE;
		uint32_t i = 0;
		while (start_len > e->matches[i].len) ++i;
		for (uint32_t len_test = start_len;; ++len_test) {
			const uint32_t cur_back = e->matches[i].dist;
			uint32_t p = normal_match_price + dist_len_price(e, cur_back, len_test, pos_state);
			if (p < opts[cur + len_test].price) {
				opts[cur + len_test].price = p; opts[cur + len_test].pos_prev = cur;
				opts[cur + len_test].back_prev = cur_back + REPS; opts[cur + len_test].prev_1_is_literal = 0;
			}
			if (len_test == e->matches[i].len) {
				/* match + literal + rep0, :729-790 */
				const uint8_t *bb = buf - cur_back - 1;
				uint32_t len_test_2 = len_test + 1;
				const uint32_t limit = buf_avail_full < len_test_2 + nice_len ? buf_avail_full : len_test_2 + nice_len;
				if (len_test_2 < limit) len_test_2 = memcmplen(buf, bb, len_test_2, limit);
				len_test_2 -= len_test + 1;
				if (len_test_2 >= 2) {
					uint32_t state_2 = st_match(state);
					uint32_t psn = (position + len_test) & e->pos_mask;
					const uint32_t calp = p + pr_bit0(e->is_match[state_2][psn])
							+ literal_price(e, position + len_test, buf[len_test - 1], 1, bb[len_test], buf[len_test]);
					state_2 = st_literal(state_2);
					psn = (psn + 1) & e->pos_mask;
					const uint32_t nrmp = calp + pr_bit1(e->is_match[state_2][psn]) + pr_bit1(e->is_rep[state_2]);
					const uint32_t offset = cur + len_test + 1 + len_test_2;
					while (len_end < offset) opts[++len_end].price = INFINITY_PRICE;
					p = nrmp + rep_price(e, 0, len_test_2, state_2, psn);
					if (p < opts[offset].price) {
						opts[offset].price = p; opts[offset].pos_prev = cur + len_test + 1; opts[offset].back_prev = 0;
						opts[offset].prev_1_is_literal = 1; opts[offset].prev_2 = 1;
						opts[offset].pos_prev_2 = cur; opts[offset].back_prev_2 = cur_back + REPS;
					}
				}
				if (++i == matches_count) break;
			}
		}
	}
	return len_end;
}

/* lzma_lzma_optimum_normal :802-858 */
static void optimum_normal(enc_t *e, mf_t *mf, uint32_t *back_res, uint32_t *len_res, uint32_t position)
{
	if (e->opts_end_index != e->opts_current_index) {
		*len_res = e->opts[e->opts_current_index].pos_prev - e->opts_current_index;
		*back_res = e->opts[e->opts_current_index].back_prev;
		e->opts_current_index = e->opts[e->opts_current_index].pos_prev;
		return;
	}
	if (mf->read_ahead == 0) {
		if (e->match_price_count >= (1 << 7)) fill_dist_prices(e);
		if (e->align_price_count >= ALIGN_SIZE) fill_align_prices(e);
	}
	uint32_t len_end = helper1(e, mf, back_res, len_res, position);
	if (len_end == UINT32_MAX) return;
	uint32_t reps[REPS];
	memcpy(reps, e->reps, sizeof(reps));
	uint32_t cur;
	for (cur = 1; cur < len_end; ++cur) {
		e->longest_match_length = mf_find(mf, &e->matches_count, e->matches);
		if (e->longest_match_length >= mf->nice_len) break;
		const uint32_t a = mf_avail(mf) + 1, b = OPTS - 1 - cur;
		len_end = helper2(e, reps, mf->buf + mf->read_pos - 1, len_end, position + cur, cur, mf->nice_len, a < b ? a : b);
	}
	backward(e, len_res, back_res, cur);
}

/* ------------------------------------------------------------------ */
/* lzma_lzma_encode, lzma/lzma_encoder.c:266-436, whole block resident */
/* (action == LZMA_FINISH from the start; SURVEY D3)                   */
/* ------------------------------------------------------------------ */
static void lzma_encode_chunk(enc_t *e, mf_t *mf, uint32_t limit)
{
	/* encode_init :266-293 */
	if (!e->is_initialized) {
		if (mf->read_pos != mf->size) {
			mf_skip(mf, 1);
			mf->read_ahead = 0;
			rc_bit(&e->rc, &e->is_match[0][0], 0);
			rc_bittree(&e->rc, e->literal + 0, 8, mf->buf[0]);
			++e->uncomp_size;
		}
		e->is_initialized = 1;
	}
	for (;;) {
		/* :343-351 */
		if (limit != UINT32_MAX && (mf->read_pos - mf->read_ahead >= limit
				|| e->rc.out_pos + rc_pending(&e->rc) >= LZMA2_CHUNK_MAX - LOOP_INPUT_MAX))
			break;
		/* :354-360 (read_limit == write_pos when finishing, lz_encoder.c:128-134) */
		if (mf->read_pos >= mf->size) {
			if (mf->read_ahead == 0) break;
		}
		uint32_t len, back;
		if (e->fast_mode) optimum_fast(e, mf, &back, &len);
		else optimum_normal(e, mf, &back, &len, (uint32_t)e->uncomp_size);
		encode_symbol(e, mf, back, len, (uint32_t)e->uncomp_size);
		e->uncomp_size += len;
	}
	rc_flush(&e->rc); /* :427-437 */
}

/* lzma2_encode, lzma/lzma2_encoder.c:134-259 with headers :53-131 */
static int lzma2_encode_block(enc_t *e, mf_t *mf, uint8_t *out, size_t out_cap, size_t *out_pos_ptr)
{
	size_t out_pos = *out_pos_ptr;
	int need_properties = 1, need_state_reset = 0, need_dictionary_reset = 1;
	int raw_with_read_ahead = 0; /* the last chunk was raw and swallowed read_ahead bytes */
	uint8_t *buf = malloc(LZMA2_HEADER_MAX + LZMA2_CHUNK_MAX);
	if (buf == NULL) return XZO_MEM_ERROR;
	int ret = XZO_OK;
	for (;;) {
		/* SEQ_INIT :146-161 */
		if (mf->size - mf->read_pos + mf->read_ahead == 0) {
			if (out_pos >= out_cap) { ret = XZO_BUF_ERROR; break; }
			out[out_pos++] = 0;
			break;
		}
		if (need_state_reset) enc_reset(e);
		size_t uncompressed_size = 0;
		/* SEQ_LZMA_ENCODE :163-214 */
		const uint32_t left = LZMA2_UNCOMPRESSED_MAX - (uint32_t)uncompressed_size;
		const uint32_t limit = mf->read_pos - mf->read_ahead + left - MATCH_LEN_MAX;
		const uint32_t read_start = mf->read_pos - mf->read_ahead;
		e->rc.out = buf + LZMA2_HEADER_MAX; e->rc.out_pos = 0;
		lzma_encode_chunk(e, mf, limit);
		size_t compressed_size = e->rc.out_pos;
		uncompressed_size += mf->read_pos - mf->read_ahead - read_start;
		if (compressed_size >= uncompressed_size) {
			/* raw chunk :202-214, header :107-131, copy mf_read lz_encoder.h:302-318 */
			if (e->ctr) { e->ctr->n_chunks_raw++; if (mf->read_ahead) e->ctr->n_raw_with_read_ahead++; }
			raw_with_read_ahead = mf->read_ahead != 0;
			uncompressed_size += mf->read_ahead;
			mf->read_ahead = 0;
			if (out_pos + 3 + uncompressed_size > out_cap) { ret = XZO_BUF_ERROR; break; }
			out[out_pos++] = need_dictionary_reset ? 1 : 2;
			need_dictionary_reset = 0;
			out[out_pos++] = (uint8_t)((uncompressed_size - 1) >> 8);
			out[out_pos++] = (uint8_t)((uncompressed_size - 1) & 0xFF);
			need_state_reset = 1;
			memcpy(out + out_pos, mf->buf + mf->read_pos - uncompressed_size, uncompressed_size);
			out_pos += uncompressed_size;
			continue;
		}
		/* lzma2_header_lzma :53-104 */
		if (e->ctr) { e->ctr->n_chunks_lzma++; e->ctr->n_raw_ahead_then_lzma += raw_with_read_ahead; }
		raw_with_read_ahead = 0;
		size_t pos;
		if (need_properties) {
			pos = 0;
			buf[pos] = need_dictionary_reset ? 0x80 + (3 << 5) : 0x80 + (2 << 5);
		} else {
			pos = 1;
			buf[pos] = need_state_reset ? 0x80 + (1 << 5) : 0x80;
		}
		const size_t buf_pos = pos;
		size_t size = uncompressed_size - 1;
		buf[pos++] += (uint8_t)(size >> 16);
		buf[pos++] = (size >> 8) & 0xFF;
		buf[pos++] = size & 0xFF;
		size = compressed_size - 1;
		buf[pos++] = (uint8_t)(size >> 8);
		buf[pos++] = size & 0xFF;
		if (need_properties) /* lzma_lzma_lclppb_encode, lzma_encoder.c:710-722 */
			buf[pos] = (uint8_t)((e->opt.pb * 5 + e->opt.lp) * 9 + e->opt.lc);
		need_properties = 0; need_state_reset = 0; need_dictionary_reset = 0;
		const size_t total = compressed_size + LZMA2_HEADER_MAX - buf_pos;
		if (out_pos + total > out_cap) { ret = XZO_BUF_ERROR; break; }
		memcpy(out + out_pos, buf + buf_pos, total);
		out_pos += total;
	}
	free(buf);
	*out_pos_ptr = out_pos;
	return ret;
}

/* ------------------------------------------------------------------ */
/* Block + Stream framing                                              */
/* ------------------------------------------------------------------ */
/* lzma_vli_encode (single call), common/vli_encoder.c:16-69 */
static size_t vli_put(uint8_t *out, uint64_t v) { size_t n = 0; while (v >= 0x80) { out[n++] = (uint8_t)v | 0x80; v >>= 7; } out[n++] = (uint8_t)v; return n; }
/* lzma_vli_size, common/vli_size.c:15-30 */
static uint32_t vli_size(uint64_t v) { uint32_t n = 0; do { v >>= 7; ++n; } while (v != 0); return n; }

static uint32_t check_size_of(uint32_t check) { return check == XZO_CHECK_NONE ? 0 : check == XZO_CHECK_CRC32 ? 4 : check == XZO_CHECK_CRC64 ? 8 : check == 10 ? 32 : UINT32_MAX; }

/* lzma2_bound + lzma_block_buffer_bound64, common/block_buffer_encoder.c:27-71 */
static uint64_t lzma2_bound(uint64_t u) { return u + ((u + LZMA2_CHUNK_MAX - 1) / LZMA2_CHUNK_MAX) * 3 + 1; }
uint64_t xzo_block_bound(uint64_t u) { return 92 + ((lzma2_bound(u) + 3) & ~(uint64_t)3); }

/* lzma_lzma2_props_encode, lzma/lzma2_encoder.c:375-400 */
static uint8_t lzma2_dict_prop(uint32_t dict_size)
{
	uint32_t d = dict_size > 4096 ? dict_size : 4096;
	--d; d |= d >> 2; d |= d >> 3; d |= d >> 4; d |= d >> 8; d |= d >> 16;
	if (d == UINT32_MAX) return 40;
	return (uint8_t)(dist_slot_of(d + 1) - 24);
}

/* lzma_block_header_size :16-68 and lzma_block_header_encode :71-131 (common/block_header_encoder.c)
 * for one LZMA2 filter with both sizes present. */
static uint32_t block_header_size(uint64_t comp, uint64_t uncomp) { return (6 + vli_size(comp) + vli_size(uncomp) + 3 + 3) & ~3u; }
static void block_header_encode(uint8_t *out, uint32_t header_size, uint64_t comp, uint64_t uncomp, uint8_t dict_prop)
{
	const size_t out_size = header_size - 4;
	out[0] = (uint8_t)(out_size / 4);
	out[1] = 0xC0; /* compressed + uncompressed size present, 1 filter */
	size_t pos = 2;
	pos += vli_put(out + pos, comp);
	pos += vli_put(out + pos, uncomp);
	out[pos++] = 0x21; out[pos++] = 0x01; out[pos++] = dict_prop; /* filter_flags_encoder.c:31-56 */
	memset(out + pos, 0, out_size - pos);
	const uint32_t crc = xzo_crc32(out, out_size, 0);
	out[out_size] = (uint8_t)crc; out[out_size + 1] = (uint8_t)(crc >> 8);
	out[out_size + 2] = (uint8_t)(crc >> 16); out[out_size + 3] = (uint8_t)(crc >> 24);
}

static size_t put_check(uint8_t *out, uint32_t check, const uint8_t *in, size_t n)
{
	if (check == XZO_CHECK_CRC32) { const uint32_t c = xzo_crc32(in, n, 0); for (int i = 0; i < 4; ++i) out[i] = (uint8_t)(c >> (8 * i)); return 4; }
	if (check == XZO_CHECK_CRC64) { const uint64_t c = xzo_crc64(in, n, 0); for (int i = 0; i < 8; ++i) out[i] = (uint8_t)(c >> (8 * i)); return 8; }
	if (check == 10) { xzo_sha256(in, n, out); return 32; } /* LZMA_CHECK_SHA256 */
	return 0;
}

/* worker_encode, common/stream_encoder_mt.c:218-359 (+ block_encoder.c:46-135 and the
 * incompressible fallback block_buffer_encoder.c:87-162, 213-281) */
/* oneshot = 0: worker_encode() framing (header size and the "does it fit" test come from
 * lzma_mt.block_size); oneshot = 1: lzma_block_buffer_encode() framing
 * (common/block_buffer_encoder.c:165-281: header size from lzma2_bound(in_size) / in_size, the LZMA2
 * data must fit lzma2_bound(in_size), else the same uncompressed fallback). */
static int block_encode_common(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint32_t check, uint64_t block_size, int oneshot, uint8_t *out, size_t *out_size_ptr,
		uint64_t *unpadded_size, xzo_counters *ctr)
{
	xzo_tables_init();
	const uint32_t csize = check_size_of(check);
	if (csize == UINT32_MAX) return XZO_UNSUPPORTED_CHECK;
	if (in_size == 0 || in_size > block_size || in_size >= (1u << 31)) return XZO_PROG_ERROR;
	size_t out_size = (size_t)xzo_block_bound(block_size); /* outbuf->allocated, :1108-1112 */
	/* :225-237: header size is computed from the MAXIMUM sizes */
	uint32_t header_size = block_header_size(out_size, block_size);
	if (oneshot) {
		header_size = block_header_size(lzma2_bound(in_size), in_size);
		out_size = header_size + (size_t)lzma2_bound(in_size); /* block_encode_normal :180-183 */
	}

	enc_t *e = malloc(sizeof(enc_t));
	if (e == NULL) return XZO_MEM_ERROR;
	int ret = enc_create(e, opt, ctr);
	if (ret != XZO_OK) { free(e); return ret; }
	mf_t mf;
	if (mf_init(&mf, in, (uint32_t)in_size, opt, ctr)) { mf_free(&mf); free(e); return XZO_MEM_ERROR; }

	size_t out_pos = header_size;
	ret = lzma2_encode_block(e, &mf, out, out_size, &out_pos);
	mf_free(&mf); free(e);
	if (ret == XZO_OK) {
		uint64_t comp = out_pos - header_size;
		const uint64_t pad = (4 - (comp & 3)) & 3;
		if (!oneshot && out_pos + pad + csize > out_size) ret = XZO_BUF_ERROR;
		else {
			for (uint64_t i = 0; i < pad; ++i) out[out_pos++] = 0; /* block_encoder.c:104-112 */
			out_pos += put_check(out + out_pos, check, in, in_size);
			block_header_encode(out, header_size, comp, in_size, lzma2_dict_prop(opt->dict_size));
			*unpadded_size = header_size + comp + csize; /* lzma_block_unpadded_size, block_util.c:53-77 */
			*out_size_ptr = out_pos;
			return XZO_OK;
		}
	}
	if (ret != XZO_BUF_ERROR) return ret;

	/* lzma_block_uncomp_encode: block_buffer_encoder.c:87-162 + :213-281 */
	const uint64_t comp = lzma2_bound(in_size);
	const uint32_t hs = block_header_size(comp, in_size);
	block_header_encode(out, hs, comp, in_size, 0x00 /* dict = LZMA_DICT_SIZE_MIN */);
	out_pos = hs;
	size_t in_pos = 0; uint8_t control = 0x01;
	while (in_pos < in_size) {
		out[out_pos++] = control; control = 0x02;
		const size_t copy = in_size - in_pos < LZMA2_CHUNK_MAX ? in_size - in_pos : LZMA2_CHUNK_MAX;
		out[out_pos++] = (uint8_t)((copy - 1) >> 8); out[out_pos++] = (uint8_t)((copy - 1) & 0xFF);
		memcpy(out + out_pos, in + in_pos, copy);
		in_pos += copy; out_pos += copy;
	}
	out[out_pos++] = 0x00;
	for (uint64_t i = comp; i & 3; ++i) out[out_pos++] = 0x00;
	out_pos += put_check(out + out_pos, check, in, in_size);
	*unpadded_size = hs + comp + csize;
	*out_size_ptr = out_pos;
	return XZO_OK;
}

int xzo_block_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint32_t check, uint64_t block_size, uint8_t *out, size_t *out_size_ptr,
		uint64_t *unpadded_size, xzo_counters *ctr)
{
	return block_encode_common(in, in_size, opt, check, block_size, 0, out, out_size_ptr, unpadded_size, ctr);
}

/* lzma_stream_header_encode / lzma_stream_footer_encode, common/stream_flags_encoder.c:29-85 */
size_t xzo_stream_header(uint8_t out[12], uint32_t check)
{
	static const uint8_t magic[6] = { 0xFD, 0x37, 0x7A, 0x58, 0x5A, 0x00 };
	memcpy(out, magic, 6);
	out[6] = 0x00; out[7] = (uint8_t)check;
	const uint32_t crc = xzo_crc32(out + 6, 2, 0);
	for (int i = 0; i < 4; ++i) out[8 + i] = (uint8_t)(crc >> (8 * i));
	return 12;
}
size_t xzo_stream_footer(uint8_t out[12], uint32_t check, uint64_t index_size)
{
	const uint32_t bs = (uint32_t)(index_size / 4 - 1);
	for (int i = 0; i < 4; ++i) out[4 + i] = (uint8_t)(bs >> (8 * i));
	out[8] = 0x00; out[9] = (uint8_t)check;
	const uint32_t crc = xzo_crc32(out + 4, 6, 0);
	for (int i = 0; i < 4; ++i) out[i] = (uint8_t)(crc >> (8 * i));
	out[10] = 'Y'; out[11] = 'Z';
	return 12;
}
/* index_encode, common/index_encoder.c:43-165; size per index.h:64-76 */
size_t xzo_index_encode(const uint64_t *unpadded, const uint64_t *uncompressed, size_t count, uint8_t *out)
{
	size_t n = 1 + vli_size(count);
	for (size_t i = 0; i < count; ++i) n += vli_size(unpadded[i]) + vli_size(uncompressed[i]);
	const size_t padded = (n + 3) & ~(size_t)3;
	if (out == NULL) return padded + 4;
	size_t pos = 0;
	out[pos++] = 0x00;
	pos += vli_put(out + pos, count);
	for (size_t i = 0; i < count; ++i) { pos += vli_put(out + pos, unpadded[i]); pos += vli_put(out + pos, uncompressed[i]); }
	while (pos < padded) out[pos++] = 0x00;
	const uint32_t crc = xzo_crc32(out, pos, 0);
	for (int i = 0; i < 4; ++i) out[pos++] = (uint8_t)(crc >> (8 * i));
	return pos;
}

size_t xzo_stream_bound(size_t in_size, uint64_t block_size)
{
	const size_t nblocks = (in_size + block_size - 1) / block_size;
	return 12 + nblocks * (size_t)xzo_block_bound(block_size) + (8 + nblocks * 18 + 8) + 12;
}

/* stream_encode_mt, common/stream_encoder_mt.c:716-888: header, blocks in order, Index, footer */
int xzo_stream_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint32_t check, uint64_t block_size, uint8_t *out, size_t out_cap,
		size_t *out_size, xzo_counters *ctr)
{
	if (out_cap < xzo_stream_bound(in_size, block_size)) return XZO_BUF_ERROR;
	const size_t nblocks = (in_size + block_size - 1) / block_size;
	uint64_t *unp = malloc((nblocks + 1) * 2 * sizeof(uint64_t));
	if (unp == NULL) return XZO_MEM_ERROR;
	uint64_t *unc = unp + nblocks + 1;
	size_t pos = xzo_stream_header(out, check);
	for (size_t b = 0; b < nblocks; ++b) {
		const size_t off = b * (size_t)block_size;
		const size_t n = in_size - off < block_size ? in_size - off : (size_t)block_size;
		size_t bs = 0;
		const int ret = xzo_block_encode(in + off, n, opt, check, block_size, out + pos, &bs, &unp[b], ctr);
		if (ret != XZO_OK) { free(unp); return ret; }
		unc[b] = n;
		pos += bs;
	}
	const size_t isz = xzo_index_encode(unp, unc, nblocks, out + pos);
	pos += isz;
	pos += xzo_stream_footer(out + pos, check, isz);
	free(unp);
	*out_size = pos;
	return XZO_OK;
}

/* MicroLZMA framing of the same LZMA core (common/microlzma_encoder.c:36-85): raw LZMA1
 * without EOPM, first output byte replaced by ~props.  Only used to pin the core against the
 * reference's single encoder known-answer test (tests/test_microlzma.c:20-32, 123-171);
 * the out_limit machinery (rc_encode_dummy) never triggers for outputs this small. */
int xzo_microlzma_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint8_t *out, size_t out_cap, size_t *out_size)
{
	xzo_tables_init();
	if (in_size == 0 || in_size > 16384 || out_cap < 65536) return XZO_BUF_ERROR;
	enc_t *e = malloc(sizeof(enc_t));
	if (e == NULL) return XZO_MEM_ERROR;
	int ret = enc_create(e, opt, NULL);
	if (ret != XZO_OK) { free(e); return ret; }
	mf_t mf;
	if (mf_init(&mf, in, (uint32_t)in_size, opt, NULL)) { mf_free(&mf); free(e); return XZO_MEM_ERROR; }
	e->rc.out = out; e->rc.out_pos = 0;
	lzma_encode_chunk(e, &mf, UINT32_MAX);
	*out_size = e->rc.out_pos;
	out[0] = (uint8_t)~((opt->pb * 5 + opt->lp) * 9 + opt->lc);
	mf_free(&mf); free(e);
	return XZO_OK;
}


/* lzma_stream_buffer_bound, common/stream_buffer_encoder.c:24-40 */
size_t xzo_stream_buffer_bound(size_t uncompressed_size) { return (size_t)xzo_block_bound(uncompressed_size) + 2 * 12 + ((1 + 1 + 2 * 9 + 4 + 3) & ~3); }

/* lzma_stream_buffer_encode (common/stream_buffer_encoder.c:43-140) == lzma_easy_buffer_encode with the
 * preset's LZMA2 options: ONE Block over the whole input via lzma_block_buffer_encode
 * (block_buffer_encoder.c:213-281).  out must hold xzo_stream_buffer_bound(in_size) (+ slack for the
 * LZMA2 attempt: the restatement encodes into a scratch first). */
int xzo_stream_buffer_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt, uint32_t check,
		uint8_t *out, size_t out_cap, size_t *out_size)
{
	if (out_cap < xzo_stream_buffer_bound(in_size)) return XZO_BUF_ERROR;
	size_t pos = xzo_stream_header(out, check);
	uint64_t unp = 0, unc = in_size;
	size_t count = 0;
	if (in_size > 0) {
		const size_t scap = (size_t)xzo_block_bound(in_size) + 70000;
		uint8_t *scratch = malloc(scap);
		if (scratch == NULL) return XZO_MEM_ERROR;
		size_t bs = 0;
		const int ret = block_encode_common(in, in_size, opt, check, in_size, 1, scratch, &bs, &unp, NULL);
		if (ret != XZO_OK) { free(scratch); return ret; }
		memcpy(out + pos, scratch, bs);
		free(scratch);
		pos += bs;
		count = 1;
	}
	const size_t isz = xzo_index_encode(&unp, &unc, count, out + pos);
	pos += isz;
	pos += xzo_stream_footer(out + pos, check, isz);
	*out_size = pos;
	return XZO_OK;
}
