// xzb_parse_warp.cuh -- warp-cooperative LZMA coder + the fast-mode parser (device only).
//
// Same decisions, bit for bit, as the sequential restatement in xzb_enc.cuh (which stays in the
// tree as the single-thread form that tests/hostsim checks against the oracle), but organised
// for one CUDA block per .xz block with every piece of coder state in shared memory.  WarpEncT is
// the part both parsers share: probability model, price tables, match store reader, symbol
// encoder, range coder and the LZMA2 chunker.  The normal-mode parser (presets 4-9) builds on it
// in xzb_parse_dp.cuh; fast mode (presets 0-3) is complete here:
//   * match lists stream from the HBM match store through a 32-position smem ring filled with
//     coalesced 16 B loads;
//   * lzma_lzma_optimum_fast needs no coder state, so its decisions are taken by a warp of their
//     own ahead of the coding warp (xzb_w_fast_parser_main);
//   * an LZMA symbol's probability indices are computed in closed form by the lanes, the
//     adaptive-probability updates happen in parallel, and only the low/range recurrence of the
//     range coder runs serially (on the coding warp, or on a coder warp: see FS).
#pragma once
#include "xzb_common.cuh"
#include "xzb_mf.cuh"
#include "xzb_frame.cuh"

#define WFULL 0xFFFFFFFFu

// flat probability layout
#define PI_IS_MATCH 0
#define PI_IS_REP 192
#define PI_IS_REP0 204
#define PI_IS_REP1 216
#define PI_IS_REP2 228
#define PI_IS_REP0_LONG 240
#define PI_DIST_SLOT 432
#define PI_DIST_SPECIAL 688
#define PI_DIST_ALIGN 802
#define PI_MATCH_LEN 818
#define PI_REP_LEN 1332
#define PI_LITERAL 1846
#define PI_TOTAL (PI_LITERAL + 0x3000)
#define LC_CHOICE 0
#define LC_CHOICE2 1
#define LC_LOW 2
#define LC_MID 130
#define LC_HIGH 258

#define XZB_MF_MARGIN 96u
#define XZB_FRING 64u
#define XZB_BACK_STALL 0xFFFFFFFEu  // ring entry: the parser warp's match-finder watchdog fired

template <class SM>
struct WarpEncT {
	static constexpr bool FAST = SM::FAST;   // fast mode: decisions come from the parser warp, nothing is priced
	SM &S;
	const uint32_t lane;
	// block + match store
	const uint8_t *buf; uint32_t size;
	const uint32_t *g_mh; const xzb_pair *g_mp; const xzb_pair *g_ovf;
	// match-finder progress: block positions [0, mf_done) are in the match store; mf_stalled = the
	// watchdog in mf_wait gave up (only the front warp polls, so the flag lives in its registers)
	const uint32_t *mf_flag; uint32_t mf_done; uint64_t mf_stall_ns;
	bool mf_stalled = false;
	uint32_t read_pos, read_ahead, ring_base;
	uint32_t f_epoch = 0, f_k = 0;  // coder warp's side of the fast-mode ring
	// params
	uint32_t nice_len, pos_mask, lc, literal_mask, dist_table_size, len_table_size, num_pos_states;
	// coder state (uniform across lanes)
	uint32_t state, rep0, rep1, rep2, rep3;
	uint32_t uncomp_size, is_initialized;
	uint32_t matches_count, longest_match_length;
	uint32_t match_price_count, align_price_count;
	uint32_t n_symbols;
	// range coder (identical in every lane)
	uint64_t rc_low; uint32_t rc_cache_size, rc_range, rc_cache, rc_out_pos; uint8_t *rc_out;
	// SM::RCQ != 0: the coded bits go through a shared-memory ring to a coder warp that runs the low/range
	// recurrence (xzb_dp_coder_main); rq_head = bits pushed so far, rq_flushes = flush markers pushed
	uint32_t rq_head = 0, rq_flushes = 0;

	__device__ WarpEncT(SM &s, uint32_t l) : S(s), lane(l) {}

	// ---------------- prices ----------------
	__device__ __forceinline__ uint32_t pr(uint32_t p, uint32_t bit) const { return S.prices[(p ^ ((0u - bit) & 2047)) >> 4]; }
	__device__ __forceinline__ uint32_t pr0(uint32_t idx) const { return S.prices[S.probs[idx] >> 4]; }
	__device__ __forceinline__ uint32_t pr1(uint32_t idx) const { return S.prices[(S.probs[idx] ^ 2047) >> 4]; }
	__device__ __forceinline__ uint32_t pr_tree(uint32_t base, uint32_t levels, uint32_t symbol) const
	{
		uint32_t price = 0; symbol += 1u << levels;
		do { const uint32_t bit = symbol & 1; symbol >>= 1; price += pr(S.probs[base + symbol], bit); } while (symbol != 1);
		return price;
	}
	__device__ __forceinline__ uint32_t pr_rtree(uint32_t base, uint32_t levels, uint32_t symbol) const
	{
		uint32_t price = 0, mi = 1;
		do { const uint32_t bit = symbol & 1; symbol >>= 1; price += pr(S.probs[base + mi], bit); mi = (mi << 1) + bit; } while (--levels != 0);
		return price;
	}

	// length_update_prices (lzma_encoder.c:76-102): one lane per table entry
	__device__ void length_update_prices(uint32_t which, uint32_t pos_state)
	{
		const uint32_t base = which ? PI_REP_LEN : PI_MATCH_LEN;
		const uint32_t a0 = pr0(base + LC_CHOICE), a1 = pr1(base + LC_CHOICE);
		const uint32_t b0 = a1 + pr0(base + LC_CHOICE2), b1 = a1 + pr1(base + LC_CHOICE2);
		for (uint32_t i = lane; i < len_table_size; i += 32) {
			uint32_t v;
			if (i < XZB_LEN_LOW) v = a0 + pr_tree(base + LC_LOW + pos_state * 8, 3, i);
			else if (i < XZB_LEN_LOW + XZB_LEN_MID) v = b0 + pr_tree(base + LC_MID + pos_state * 8, 3, i - XZB_LEN_LOW);
			else v = b1 + pr_tree(base + LC_HIGH, 8, i - XZB_LEN_LOW - XZB_LEN_MID);
			S.len_prices[which][pos_state][i] = v;
		}
		if (lane == 0) S.len_counters[which][pos_state] = len_table_size;
		__syncwarp();
	}

	// fill_dist_prices / fill_align_prices (lzma_encoder_optimum_normal.c:131-195)
	__device__ void fill_dist_prices()
	{
		for (uint32_t t = lane; t < XZB_DIST_STATES * dist_table_size; t += 32) {
			const uint32_t ds = t / dist_table_size, s = t - ds * dist_table_size;
			uint32_t v = pr_tree(PI_DIST_SLOT + ds * 64, 6, s);
			if (s >= XZB_DIST_MODEL_END) v += (((s >> 1) - 1) - XZB_ALIGN_BITS) << 4;
			S.dist_slot_prices[ds][s] = v;
		}
		__syncwarp();
		for (uint32_t i = lane; i < XZB_FULL_DISTANCES; i += 32) {
			if (i < XZB_DIST_MODEL_START) {
				for (uint32_t ds = 0; ds < XZB_DIST_STATES; ++ds) S.dist_prices[ds][i] = S.dist_slot_prices[ds][i];
			} else {
				const uint32_t slot = xzb_dist_slot(i);
				const uint32_t footer_bits = (slot >> 1) - 1;
				const uint32_t base = (2 | (slot & 1)) << footer_bits;
				const uint32_t price = pr_rtree(PI_DIST_SPECIAL + base - slot - 1, footer_bits, i - base);
				for (uint32_t ds = 0; ds < XZB_DIST_STATES; ++ds) S.dist_prices[ds][i] = price + S.dist_slot_prices[ds][slot];
			}
		}
		match_price_count = 0;
		__syncwarp();
	}
	__device__ void fill_align_prices()
	{
		if (lane < XZB_ALIGN_SIZE) S.align_prices[lane] = pr_rtree(PI_DIST_ALIGN, XZB_ALIGN_BITS, lane);
		align_price_count = 0;
		__syncwarp();
	}

	// lzma_lzma_encoder_reset (lzma_encoder.c:528-598)
	__device__ void reset()
	{
		for (uint32_t i = lane; i < PI_TOTAL; i += 32) S.probs[i] = 1024;
		__syncwarp();
		rc_low = 0; rc_cache_size = 1; rc_range = 0xFFFFFFFFu; rc_cache = 0;
		state = 0; rep0 = rep1 = rep2 = rep3 = 0;
		if constexpr (!FAST)
			for (uint32_t w = 0; w < 2; ++w)
				for (uint32_t ps = 0; ps < num_pos_states; ++ps) length_update_prices(w, ps);
		match_price_count = 0xFFFFFFFFu / 2;
		align_price_count = 0xFFFFFFFFu / 2;
	}

	// ---------------- match store reader ----------------
	__device__ __forceinline__ uint32_t mf_avail() const { return size - read_pos; }

	// The binary-tree match finder publishes its progress segment by segment while this kernel runs
	// (xzb_k_publish).  Only this warp polls; at a refill it asks for XZB_MF_MARGIN positions beyond
	// the refill's first position.  Segment boundaries are multiples of 256 positions, so a cache line of
	// mh/mp never mixes finished and unfinished rows; the overflow pool is read past L1 (__ldcg).
	__device__ __forceinline__ void mf_wait(uint32_t need)
	{
		uint64_t t0 = 0;
		uint32_t last = mf_done;
		for (;;) {
			uint32_t d = 0;
			if (lane == 0) asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(d) : "l"(mf_flag) : "memory");
			d = __shfl_sync(WFULL, d, 0);
			if (d >= need) { mf_done = d; return; }
			uint64_t now;
			asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
			now = __shfl_sync(WFULL, now, 0);
			if (t0 == 0 || d != last) { last = d; t0 = now; }
			else if (now - t0 > mf_stall_ns) {  // watchdog: give the block up, the host parses again later
				mf_done = 0xFFFFFFFFu;
				mf_stalled = true;
				return;
			}
			__nanosleep(2000);
		}
	}

	// Fill S.m_* with the match list of block position p (ring refill as needed); returns the header word.
	__device__ uint32_t mf_load(uint32_t p)
	{
		if (p - ring_base >= 32u) {  // refill: 32 consecutive positions, one per lane (coalesced 64 B each)
			__syncwarp();
			ring_base = p;
			const uint32_t need = xzb_min(p + XZB_MF_MARGIN, size);
			if (need > mf_done) mf_wait(need);
			const uint32_t g = p + lane;
			if (mf_stalled) {
				S.ring_mh[lane] = 0;  // "no matches": keeps every later step in bounds until the chunk loop exits
			} else if (g < size) {
				S.ring_mh[lane] = g_mh[g];
				const uint4 *src = reinterpret_cast<const uint4 *>(g_mp + (size_t)g * 8);
				uint4 *dst = reinterpret_cast<uint4 *>(&S.ring_mp[lane][0]);
				const uint4 a = src[0], b = src[1], c = src[2], d = src[3];
				dst[0] = a; dst[1] = b; dst[2] = c; dst[3] = d;
			}
			__syncwarp();
		}
		const uint32_t slot = p - ring_base;
		const uint32_t h = S.ring_mh[slot];
		const uint32_t count = h & 0xFFFF;
		__syncwarp();  // previous users of S.m_* are done
		if (count <= 8) {
			if (lane < count) put_match(lane, S.ring_mp[slot][lane]);
		} else {
			if (lane < 7) put_match(lane, S.ring_mp[slot][lane]);
			const xzb_pair *o = g_ovf + S.ring_mp[slot][7].len;
			for (uint32_t i = 7 + lane; i < count; i += 32) {
				const uint2 v = __ldcg(reinterpret_cast<const uint2 *>(o + (i - 7)));
				put_match(i, xzb_pair{ v.x, v.y });
			}
		}
		__syncwarp();
		return h;
	}

	__device__ uint32_t mf_find(uint32_t *count_ptr)  // lzma_mf_find semantics on the match store
	{
		const uint32_t h = mf_load(read_pos);
		*count_ptr = h & 0xFFFF;
		++read_pos; ++read_ahead;
		return h >> 16;
	}
	__device__ __forceinline__ void put_match(uint32_t i, const xzb_pair v)
	{
		S.m_len[i] = (uint16_t)XZB_PAIR_LEN(v.len); S.m_len2[i] = (uint16_t)XZB_PAIR_LEN2(v.len);
		S.m_mb[i] = (uint8_t)XZB_PAIR_MB(v.len); S.m_dist[i] = v.dist;
	}
	__device__ __forceinline__ void mf_skip(uint32_t amount) { read_pos += amount; read_ahead += amount; }

	// lzma_memcmplen: first index >= len where a and b differ, capped at limit (uniform args)
	__device__ uint32_t memcmplen(const uint8_t *a, const uint8_t *b, uint32_t len, uint32_t limit) const
	{
		while (len < limit) {
			const uint32_t j = len + lane;
			const bool ne = (j < limit) ? (a[j] != b[j]) : true;
			const uint32_t m = __ballot_sync(WFULL, ne);
			if (m != 0) return len + (uint32_t)__ffs((int)m) - 1;
			len += 32;
		}
		return len;
	}

	// memcmplen(a, b, start, limit_true) given `mg` = bit j set iff (j >= limit_m || a[j] != b[j]) for j = 0..7,
	// where bytes [0, start) are known equal and limit_m <= limit_true.  Touches memory only when the
	// answer lies beyond the eight bytes already compared.
	__device__ __forceinline__ uint32_t mlen_from(uint32_t mg, uint32_t start, uint32_t limit_m, const uint8_t *a, const uint8_t *b, uint32_t limit_true) const
	{
		if (start >= limit_true) return start;
		if (start < 8) {
			const uint32_t hi = mg >> start;
			if (hi != 0) {
				const uint32_t f = start + (uint32_t)__ffs((int)hi) - 1;
				if (f < limit_m) return f;            // genuine mismatch
				return memcmplen(a, b, f, limit_true);  // f == limit_m: the mask stopped there, the data may go on
			}
			return memcmplen(a, b, 8, limit_true);
		}
		return memcmplen(a, b, start, limit_true);
	}

	// lengths of the four rep matches at buf (0 when the first two bytes differ), limit >= 2:
	// one round of loads, lane = (rep index, byte 0..7); longer matches continue in mlen_from
	__device__ void rep_lens4(const uint8_t *b, uint32_t limit, uint32_t out[4]) const
	{
		const uint32_t j = lane & 7;
		const uint32_t rr = rep_of(lane >> 3);
		const bool in = j < limit;
		const uint32_t av = in ? b[j] : 0u, cv = in ? (b - rr - 1)[j] : 0x100u;
		const uint32_t m = __ballot_sync(WFULL, av != cv);
#pragma unroll
		for (uint32_t r = 0; r < 4; ++r) {
			const uint32_t mg = (m >> (8 * r)) & 0xFF;
			out[r] = (mg & 3) ? 0u : mlen_from(mg, 2, limit, b, b - rep_of(r) - 1, limit);
		}
	}

	// get_literal_price (lzma_encoder_optimum_normal.c:20-53): one lane per tree level
	__device__ uint32_t literal_price(uint32_t pos, uint32_t prev_byte, bool match_mode, uint32_t match_byte, uint32_t symbol) const
	{
		const uint32_t sub = PI_LITERAL + 3u * ((((pos << 8) + prev_byte) & literal_mask) << lc);
		uint32_t v = 0;
		if (lane < 8) {
			const uint32_t i = lane;
			const uint32_t pre = (symbol | 0x100) >> (8 - i);
			const uint32_t bit = (symbol >> (7 - i)) & 1;
			uint32_t idx = pre;
			if (match_mode) {
				const uint32_t off = ((symbol ^ match_byte) >> (8 - i)) == 0 ? 0x100u : 0u;
				const uint32_t mbit = ((match_byte >> (7 - i)) & 1) ? off : 0u;
				idx = off + mbit + pre;
			}
			v = pr(S.probs[sub + idx], bit);
		}
		return __reduce_add_sync(WFULL, v);
	}

	// matched-mode literal price computed by ONE lane (every lane may price a different literal)
	__device__ __forceinline__ uint32_t literal_price_matched_lane(uint32_t pos, uint32_t prev_byte, uint32_t match_byte, uint32_t symbol) const
	{
		const uint32_t sub = PI_LITERAL + 3u * ((((pos << 8) + prev_byte) & literal_mask) << lc);
		uint32_t price = 0, offset = 0x100;
		symbol += 1u << 8;
		do {
			match_byte <<= 1;
			const uint32_t match_bit = match_byte & offset;
			const uint32_t idx = offset + match_bit + (symbol >> 8);
			const uint32_t bit = (symbol >> 7) & 1;
			price += pr(S.probs[sub + idx], bit);
			symbol <<= 1;
			offset &= ~(match_byte ^ symbol);
		} while (symbol < (1u << 16));
		return price;
	}

	__device__ __forceinline__ uint32_t len_price(uint32_t which, uint32_t len, uint32_t ps) const { return S.len_prices[which][ps][len - XZB_MATCH_LEN_MIN]; }
	__device__ __forceinline__ uint32_t short_rep_price(uint32_t st, uint32_t ps) const { return pr0(PI_IS_REP0 + st) + pr0(PI_IS_REP0_LONG + (st << 4) + ps); }
	__device__ __forceinline__ uint32_t pure_rep_price(uint32_t rep, uint32_t st, uint32_t ps) const
	{
		if (rep == 0) return pr0(PI_IS_REP0 + st) + pr1(PI_IS_REP0_LONG + (st << 4) + ps);
		uint32_t price = pr1(PI_IS_REP0 + st);
		if (rep == 1) price += pr0(PI_IS_REP1 + st);
		else { price += pr1(PI_IS_REP1 + st); price += pr(S.probs[PI_IS_REP2 + st], rep - 2); }
		return price;
	}
	__device__ __forceinline__ uint32_t rep_price(uint32_t rep, uint32_t len, uint32_t st, uint32_t ps) const { return len_price(1, len, ps) + pure_rep_price(rep, st, ps); }
	__device__ __forceinline__ uint32_t dist_len_price(uint32_t dist, uint32_t len, uint32_t ps) const
	{
		const uint32_t ds = xzb_dist_state(len);
		uint32_t price;
		if (dist < XZB_FULL_DISTANCES) price = S.dist_prices[ds][dist];
		else price = S.dist_slot_prices[ds][xzb_dist_slot(dist)] + S.align_prices[dist & XZB_ALIGN_MASK];
		return price + len_price(0, len, ps);
	}

	// ---------------- range coder ----------------
	// The range coder state is kept identical in all lanes (every lane runs the recurrence); only
	// lane 0 stores the output bytes.  range_encoder.h:135-159
	__device__ __forceinline__ void rc_shift_low()
	{
		if ((uint32_t)rc_low < 0xFF000000u || (uint32_t)(rc_low >> 32) != 0) {
			const uint8_t carry = (uint8_t)(rc_low >> 32);
			uint8_t c = (uint8_t)rc_cache;
			do {
				if (lane == 0) rc_out[rc_out_pos] = (uint8_t)(c + carry);
				++rc_out_pos;
				c = 0xFF;
			} while (--rc_cache_size != 0);
			rc_cache = (uint32_t)((rc_low >> 24) & 0xFF);
		}
		++rc_cache_size;
		rc_low = (rc_low & 0x00FFFFFF) << 8;
	}

	// one coded bit: p = probability before adaptation, 0xFFFF = direct bit (range_encoder.h:196-234)
	__device__ __forceinline__ void rc_step(uint32_t p, uint32_t bit)
	{
		if (rc_range < (1u << 24)) { rc_shift_low(); rc_range <<= 8; }
		if (p == 0xFFFF) {
			rc_range >>= 1;
			if (bit) rc_low += rc_range;
		} else {
			const uint32_t bound = (rc_range >> 11) * p;
			if (bit) { rc_low += bound; rc_range -= bound; } else rc_range = bound;
		}
	}

	// the same for a bit that is known to be probability-coded (no direct-bit test on the chain)
	__device__ __forceinline__ void rc_step_prob(uint32_t p, uint32_t bit)
	{
		if (rc_range < (1u << 24)) { rc_shift_low(); rc_range <<= 8; }
		const uint32_t bound = (rc_range >> 11) * p;
		rc_low += bit ? bound : 0u;
		rc_range = bit ? rc_range - bound : bound;
	}

	__device__ void rc_flush()  // rc_flush + RC_FLUSH handling, range_encoder.h:127-132, 198-203, 236-249
	{
		if constexpr (SM::RCQ != 0) {   // marker record; the coder warp flushes, then reports the chunk's size
			__syncwarp();
			if (lane == 0) {
				S.rcq[rq_head & (SM::RCQ - 1)] = 0x8000;
				asm volatile("" ::: "memory");
				S.rcq_head = rq_head + 1;
			}
			++rq_head; ++rq_flushes;
			while (S.rcq_flushes != rq_flushes) { }
			asm volatile("" ::: "memory");
			rc_out_pos = S.rcq_out_pos;
			__syncwarp();
			return;
		}
		rc_flush_local();
	}
	__device__ __forceinline__ void set_rc_out(uint8_t *p)   // start of a chunk's range coder output
	{
		rc_out = p; rc_out_pos = 0;
		if constexpr (SM::RCQ != 0) { if (lane == 0) S.rcq_out = p; __syncwarp(); }
	}
	__device__ void rc_flush_local()
	{
		if (rc_range < (1u << 24)) { rc_shift_low(); rc_range <<= 8; }
		for (int i = 0; i < 5; ++i) rc_shift_low();
		rc_low = 0; rc_cache_size = 1; rc_range = 0xFFFFFFFFu; rc_cache = 0;
		__syncwarp();
	}

	// ---- one symbol's bits: resolved by the lanes in closed form, coded from a shared-memory list ----
	// The low/range recurrence (range_encoder.h:196-234) is the only serial part of a symbol.  The lanes
	// put (probability before adaptation | bit << 12 | direct-bit flag << 13) of "their" bit into
	// S.rc_bits and adapt the probability; rc_run then walks the list with the loads issued four
	// bits ahead of their use (they do not depend on the recurrence), every lane running the same
	// recurrence so that low/range stay uniform.
	__device__ __forceinline__ void rc_put(uint32_t k, uint32_t idx, uint32_t bit)   // probability-coded bit k
	{
		const uint32_t pv = S.probs[idx];
		S.probs[idx] = (xzb_prob)(bit ? pv - (pv >> 5) : pv + ((2048 - pv) >> 5));
		if constexpr (SM::RCQ != 0) S.rcq[(rq_head + k) & (SM::RCQ - 1)] = (uint16_t)(pv | (bit << 12));
		else S.rc_bits[k] = (uint16_t)(pv | (bit << 12));
	}
	__device__ __forceinline__ void rc_put_direct(uint32_t k, uint32_t bit)   // direct bit k (rc_direct, range_encoder.h:111-119)
	{
		if constexpr (SM::RCQ != 0) S.rcq[(rq_head + k) & (SM::RCQ - 1)] = (uint16_t)(0x2000u | (bit << 12));
		else S.rc_bits[k] = (uint16_t)(0x2000u | (bit << 12));
	}
	// "*out_pos + rc_pending() >= limit" of the chunk loop (lzma_encoder.c:325-331).  out_pos + pending = 1 + the number
	// of normalisation shifts so far; with the coder warp behind by q bits it is at most its published value + q
	// (one shift per bit at most), so the exact value is only waited for within the last few bytes of a chunk.
	__device__ __forceinline__ bool rc_pending_reaches(uint32_t limit)
	{
		if constexpr (SM::RCQ != 0) {
			for (;;) {
				const uint32_t tail = S.rcq_tail;
				asm volatile("" ::: "memory");
				const uint32_t T = S.rcq_T;
				if (T + (rq_head - tail) + 4 < limit) return false;
				if (tail == rq_head) return T + 4 >= limit;
			}
		}
		return rc_out_pos + (rc_cache_size + 4) >= limit;
	}
	// Two passes over at most 32 bits at a time.  Pass 1 is the range recurrence alone, branch-free: whether a
	// normalisation shift precedes the bit and what the bit adds to `low` are captured by lane k for bit k.
	// Pass 2 applies the additions to `low` segment by segment between the (few) shifts, taking the segment sums
	// from a warp prefix sum, so rc_shift_low -- the only branchy part -- runs once per shift, not once per bit.
	__device__ __forceinline__ void rc_run32(uint32_t first, uint32_t m)
	{
		const uint2 *B = reinterpret_cast<const uint2 *>(S.rc_bits + first);   // first is a multiple of 32
		uint32_t range = rc_range;
		uint32_t my_add = 0; bool my_need = false;
		uint2 v = B[0];
		for (uint32_t i = 0; i < m; i += 4) {
			const uint2 c = v;
			v = B[(i >> 2) + 1];   // rc_bits has room for the read past the end
#pragma unroll
			for (uint32_t u = 0; u < 4; ++u) {
				const uint32_t w = u == 0 ? (c.x & 0xFFFF) : u == 1 ? (c.x >> 16) : u == 2 ? (c.y & 0xFFFF) : (c.y >> 16);
				const bool live = i + u < m;
				const bool need = live && range < (1u << 24);
				range = need ? range << 8 : range;
				const uint32_t bit = (w >> 12) & 1;
				const bool isd = (w & 0x2000) != 0;
				const uint32_t half = range >> 1;
				const uint32_t bound = (range >> 11) * (w & 0xFFF);
				const uint32_t add = bit ? (isd ? half : bound) : 0u;
				const uint32_t nr = isd ? half : (bit ? range - bound : bound);
				range = live ? nr : range;
				if (lane == i + u) { my_add = live ? add : 0u; my_need = need; }
			}
		}
		rc_range = range;
		// inclusive prefix sums of the additions (64 bit: up to 32 x 2^32)
		unsigned long long ps = my_add;
#pragma unroll
		for (uint32_t d = 1; d < 32; d <<= 1) {
			const unsigned long long o = __shfl_up_sync(WFULL, ps, d);
			if (lane >= d) ps += o;
		}
		uint32_t mask = __ballot_sync(WFULL, my_need);
		unsigned long long done = 0;
		while (mask) {
			const uint32_t j = (uint32_t)__ffs((int)mask) - 1;   // a shift precedes bit j: bits before j go in first
			mask &= mask - 1;
			const unsigned long long upto = j ? __shfl_sync(WFULL, ps, j - 1) : 0ull;
			rc_low += upto - done;
			done = upto;
			rc_shift_low();
		}
		rc_low += __shfl_sync(WFULL, ps, 31) - done;
	}
	__device__ void rc_run(uint32_t n)
	{
		__syncwarp();
		if constexpr (SM::RCQ != 0) {   // publish the symbol's bits to the coder warp
			rq_head += n;
			asm volatile("" ::: "memory");
			if (lane == 0) S.rcq_head = rq_head;
			return;
		}
		rc_run32(0, n < 32 ? n : 32);
		if (n > 32) rc_run32(32, n - 32);
		__syncwarp();
	}
	// bit j of an nbits-wide value coded MSB first through a bit tree at `base` (rc_bittree, range_encoder.h:86-95)
	static __device__ __forceinline__ void bt_at(uint32_t base, uint32_t nbits, uint32_t v, uint32_t j, uint32_t &idx, uint32_t &bit)
	{
		idx = base + ((1u << j) | (v >> (nbits - j)));
		bit = (v >> (nbits - 1 - j)) & 1;
	}
	// bit j of a value coded LSB first (rc_bittree_reverse, :98-108): the node index is 1 followed by the bits so far
	static __device__ __forceinline__ void rt_at(uint32_t base, uint32_t v, uint32_t j, uint32_t &idx, uint32_t &bit)
	{
		idx = base + ((1u << j) | (j ? (__brev(v) >> (32 - j)) : 0u));
		bit = (v >> j) & 1;
	}
	// the length price bookkeeping of length() (lzma_encoder.c:105-134): the refresh must see the probabilities
	// from before this length's own bits (DESIGN.md F2)
	__device__ __forceinline__ void length_count(uint32_t which, uint32_t pos_state)
	{
		if constexpr (!FAST) {
			const uint32_t c = S.len_counters[which][pos_state] - 1;
			__syncwarp();
			if (c == 0) length_update_prices(which, pos_state);
			else { if (lane == 0) S.len_counters[which][pos_state] = c; __syncwarp(); }
		}
	}
	// Lane k's bit of "prefix bits, then a length, then (matches) a distance".  pre_n prefix bits are given by
	// (pre_idx, pre_bit) of lane k < pre_n; dist == 0xFFFFFFFF: no distance (rep match).
	__device__ void encode_len_dist(uint32_t pre_n, uint32_t pre_idx, uint32_t pre_bit, uint32_t which, uint32_t pos_state, uint32_t len, uint32_t dist)
	{
		const uint32_t lbase = which ? PI_REP_LEN : PI_MATCH_LEN;
		const uint32_t lenx = len - XZB_MATCH_LEN_MIN;
		uint32_t nch, tb, tbits, lv;   // choice bits, the tree, its depth, the value in it
		if (lenx < XZB_LEN_LOW) { nch = 1; tb = lbase + LC_LOW + pos_state * 8; tbits = 3; lv = lenx; }
		else if (lenx < XZB_LEN_LOW + XZB_LEN_MID) { nch = 2; tb = lbase + LC_MID + pos_state * 8; tbits = 3; lv = lenx - XZB_LEN_LOW; }
		else { nch = 2; tb = lbase + LC_HIGH; tbits = 8; lv = lenx - XZB_LEN_LOW - XZB_LEN_MID; }
		const uint32_t o1 = pre_n, o2 = o1 + nch, o3 = o2 + tbits;
		uint32_t n = o3, slot = 0, fb = 0, dbase = 0, reduced = 0, nd = 0, o4 = o3;
		if (dist != 0xFFFFFFFFu) {
			slot = xzb_dist_slot(dist);
			o4 = o3 + 6; n = o4;
			if (slot >= XZB_DIST_MODEL_START) {
				fb = (slot >> 1) - 1;
				dbase = (2 | (slot & 1)) << fb;
				reduced = dist - dbase;
				nd = slot < XZB_DIST_MODEL_END ? 0 : fb - XZB_ALIGN_BITS;
				n = o4 + fb;
			}
		}
		const uint32_t dsb = PI_DIST_SLOT + xzb_dist_state(len) * 64;
#pragma unroll
		for (uint32_t rnd = 0; rnd < 2; ++rnd) {
			const uint32_t k = lane + 32 * rnd;
			if (k < n) {
				uint32_t idx = 0, bit = 0;
				bool direct = false;
				if (k < o1) { idx = pre_idx; bit = pre_bit; }
				else if (k < o2) { const uint32_t j = k - o1; idx = lbase + (j == 0 ? LC_CHOICE : LC_CHOICE2); bit = j == 0 ? (lenx >= XZB_LEN_LOW) : (lenx >= XZB_LEN_LOW + XZB_LEN_MID); }
				else if (k < o3) bt_at(tb, tbits, lv, k - o2, idx, bit);
				else if (k < o4) bt_at(dsb, 6, slot, k - o3, idx, bit);
				else if (nd == 0 && slot < XZB_DIST_MODEL_END) rt_at(PI_DIST_SPECIAL + dbase - slot - 1, reduced, k - o4, idx, bit);
				else if (k - o4 < nd) { direct = true; bit = ((reduced >> XZB_ALIGN_BITS) >> (nd - 1 - (k - o4))) & 1; }
				else rt_at(PI_DIST_ALIGN, reduced & XZB_ALIGN_MASK, k - o4 - nd, idx, bit);
				if (direct) rc_put_direct(k, bit);
				else rc_put(k, idx, bit);
			}
		}
		rc_run(n);
	}

	// Literal fast path of encode_symbol (lzma_encoder.c:22-69, 240-246): lane 0 = is_match bit,
	// lanes 1..8 = the eight tree levels.
	__device__ void encode_literal(uint32_t position)
	{
		const uint32_t pos_state = position & pos_mask;
		++n_symbols;
		const uint32_t p = read_pos - read_ahead;
		const uint32_t cur_byte = buf[p];
		const uint32_t sub = PI_LITERAL + 3u * ((((position << 8) + buf[p - 1]) & literal_mask) << lc);
		const bool matched = state >= XZB_LIT_STATES;
		const uint32_t mb = matched ? buf[p - rep0 - 1] : 0;
		uint32_t idx = 0, bit = 0;
		if (lane == 0) {
			idx = PI_IS_MATCH + (state << 4) + pos_state;
		} else if (lane < 9) {
			const uint32_t j = lane - 1;
			const uint32_t pre = (cur_byte | 0x100) >> (8 - j);
			bit = (cur_byte >> (7 - j)) & 1;
			idx = sub + pre;
			if (matched) {
				const uint32_t off = ((cur_byte ^ mb) >> (8 - j)) == 0 ? 0x100u : 0u;
				const uint32_t mbit = ((mb >> (7 - j)) & 1) ? off : 0u;
				idx = sub + off + mbit + pre;
			}
		}
		if (lane < 9) rc_put(lane, idx, bit);
		state = matched ? (state <= 9 ? state - 3 : state - 6) : (state <= 3 ? 0 : state - 3);
		rc_run(9);
		read_ahead -= 1;
	}

	// encode_symbol (lzma_encoder.c:232-263): literal (:22-69), match (:152-175), rep_match (:178-229)
	__device__ void encode_symbol(uint32_t back, uint32_t len, uint32_t position)
	{
		if (back == XZB_BACK_LITERAL) { encode_literal(position); return; }
		const uint32_t pos_state = position & pos_mask;
		++n_symbols;
		const uint32_t st = state;
		if (back >= XZB_REPS) {   // match: is_match 1, is_rep 0, length, distance
			const uint32_t distance = back - XZB_REPS;
			length_count(0, pos_state);
			const uint32_t pidx = lane == 0 ? PI_IS_MATCH + (st << 4) + pos_state : PI_IS_REP + st;
			encode_len_dist(2, pidx, lane == 0 ? 1u : 0u, 0, pos_state, len, distance);
			state = st < XZB_LIT_STATES ? 7 : 10;
			if (xzb_dist_slot(distance) >= XZB_DIST_MODEL_END) ++align_price_count;
			rep3 = rep2; rep2 = rep1; rep1 = rep0; rep0 = distance;
			++match_price_count;
		} else {                  // rep match: is_match 1, is_rep 1, is_rep0 / is_rep0_long / is_rep1 / is_rep2, length
			uint32_t pre_n, pidx, pbit;
			if (back == 0) {
				pre_n = 4;
				pidx = lane == 0 ? PI_IS_MATCH + (st << 4) + pos_state : lane == 1 ? PI_IS_REP + st : lane == 2 ? PI_IS_REP0 + st : PI_IS_REP0_LONG + (st << 4) + pos_state;
				pbit = lane < 2 ? 1u : lane == 2 ? 0u : (len != 1 ? 1u : 0u);
			} else {
				pre_n = back == 1 ? 4 : 5;
				pidx = lane == 0 ? PI_IS_MATCH + (st << 4) + pos_state : lane == 1 ? PI_IS_REP + st : lane == 2 ? PI_IS_REP0 + st : lane == 3 ? PI_IS_REP1 + st : PI_IS_REP2 + st;
				pbit = lane < 3 ? 1u : lane == 3 ? (back == 1 ? 0u : 1u) : back - 2;
				uint32_t distance;
				if (back == 1) distance = rep1;
				else { if (back == 3) { distance = rep3; rep3 = rep2; } else distance = rep2; rep2 = rep1; }
				rep1 = rep0; rep0 = distance;
			}
			if (len == 1) {           // short rep: the prefix bits only
				if (lane < pre_n) rc_put(lane, pidx, pbit);
				rc_run(pre_n);
				state = st < XZB_LIT_STATES ? 9 : 11;
			} else {
				length_count(1, pos_state);
				encode_len_dist(pre_n, pidx, pbit, 1, pos_state, len, 0xFFFFFFFFu);
				state = st < XZB_LIT_STATES ? 8 : 11;
			}
		}
		read_ahead -= len;
	}

	__device__ __forceinline__ uint32_t rep_of(uint32_t i) const { return i == 0 ? rep0 : i == 1 ? rep1 : i == 2 ? rep2 : rep3; }

	// ---------------- lzma_lzma_optimum_fast (lzma_encoder_optimum_fast.c:19-169) ----------------
	__device__ void optimum_fast(uint32_t *back_res, uint32_t *len_res)
	{
		uint32_t len_main, mcount;
		if (read_ahead == 0) {
			len_main = mf_find(&mcount);
		} else {
			len_main = longest_match_length;
			mcount = matches_count;
		}
		const uint8_t *b = buf + read_pos - 1;
		const uint32_t buf_avail = xzb_min(mf_avail() + 1, XZB_MATCH_LEN_MAX);
		if (buf_avail < 2) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return; }
		uint32_t rl[4];
		rep_lens4(b, buf_avail, rl);
		uint32_t rep_len = 0, rep_index = 0;
		for (uint32_t i = 0; i < XZB_REPS; ++i) {
			if (rl[i] == 0) continue;
			if (rl[i] >= nice_len) { *back_res = i; *len_res = rl[i]; mf_skip(rl[i] - 1); return; }
			if (rl[i] > rep_len) { rep_index = i; rep_len = rl[i]; }
		}
		if (len_main >= nice_len) {
			*back_res = S.m_dist[mcount - 1] + XZB_REPS; *len_res = len_main;
			mf_skip(len_main - 1); return;
		}
		uint32_t back_main = 0;
		if (len_main >= 2) {
			back_main = S.m_dist[mcount - 1];
			while (mcount > 1 && len_main == S.m_len[mcount - 2] + 1) {
				if (!xzb_change_pair_w(S.m_dist[mcount - 2], back_main)) break;
				--mcount;
				len_main = S.m_len[mcount - 1];
				back_main = S.m_dist[mcount - 1];
			}
			if (len_main == 2 && back_main >= 0x80) len_main = 1;
		}
		if (rep_len >= 2) {
			if (rep_len + 1 >= len_main || (rep_len + 2 >= len_main && back_main > (1u << 9))
					|| (rep_len + 3 >= len_main && back_main > (1u << 15))) {
				*back_res = rep_index; *len_res = rep_len; mf_skip(rep_len - 1); return;
			}
		}
		if (len_main < 2 || buf_avail <= 2) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return; }
		longest_match_length = mf_find(&matches_count);
		if (longest_match_length >= 2) {
			const uint32_t new_dist = S.m_dist[matches_count - 1];
			if ((longest_match_length >= len_main && new_dist < back_main)
					|| (longest_match_length == len_main + 1 && !xzb_change_pair_w(back_main, new_dist))
					|| (longest_match_length > len_main + 1)
					|| (longest_match_length + 1 >= len_main && len_main >= 3 && xzb_change_pair_w(new_dist, back_main))) {
				*back_res = XZB_BACK_LITERAL; *len_res = 1; return;
			}
		}
		++b;
		const uint32_t limit = xzb_max(2, len_main - 1);
		for (uint32_t i = 0; i < XZB_REPS; ++i) {
			if (memcmplen(b, b - rep_of(i) - 1, 0, limit) == limit) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return; }
		}
		*back_res = back_main + XZB_REPS; *len_res = len_main;
		mf_skip(len_main - 2);
	}
	static __device__ __forceinline__ bool xzb_change_pair_w(uint32_t small_dist, uint32_t big_dist) { return (big_dist >> 7) > small_dist; }

	// index of the first match whose len >= l (matches sorted by len); uniform or per-lane
	__device__ __forceinline__ uint32_t match_index_for(uint32_t l, uint32_t mcount) const
	{
		uint32_t i = 0;
		while (i + 1 < mcount && S.m_len[i] < l) ++i;
		return i;
	}

	// ---------------- fast mode: decisions come from the parser warp (xzb_w_fast_parser_main) ----------------
	// Every entry carries read_pos / read_ahead as they were right after lzma_lzma_optimum_fast returned,
	// so this warp sees exactly the values the sequential encoder would have at every chunk decision.
	__device__ __forceinline__ void fast_pop(uint32_t *back, uint32_t *len)
	{
		const uint32_t slot = f_k % XZB_FRING;
		const uint64_t want = ((uint64_t)f_epoch << 32) | (uint64_t)(f_k + 1);
		while (S.f_tag[slot] != want) { }
		asm volatile("" ::: "memory");   // shared-memory loads issue in order behind the tag (no fence.cta: see DP_RELEASE in xzb_parse_dp.cuh)
		const uint32_t lr = S.f_lenra[slot];
		*back = S.f_back[slot];
		*len = lr & 0xFFFF;
		read_pos = S.f_rpos[slot];
		read_ahead = lr >> 16;
		++f_k;
		__syncwarp();
		if (lane == 0) S.f_consumed = f_k;
	}
	// (re)start the parser warp at block position pos with reps = 0: at the first symbol and after an
	// uncompressed chunk (lzma2_encoder.c:228-236 clears read_ahead and asks for a state reset)
	__device__ __forceinline__ void fast_restart(uint32_t pos)
	{
		f_k = 0; ++f_epoch;
		__syncwarp();
		if (lane == 0) { S.f_consumed = 0; S.f_start_pos = pos; __threadfence_block(); S.f_epoch = f_epoch; }
		__syncwarp();
	}

	// ---------------- lzma_lzma_encode for one LZMA2 chunk (lzma_encoder.c:266-436), fast mode ----------------
	// (normal mode: DpEnc::encode_chunk)
	__device__ void encode_chunk(uint32_t limit)
	{
		if (!is_initialized) {
			if (read_pos != size) {
				mf_skip(1);
				read_ahead = 0;
				// lzma_encoder.c:296-303: is_match[0][0] = 0, then the byte through literal coder 0
				if (lane < 9) {
					uint32_t idx = PI_IS_MATCH, bit = 0;
					if (lane) bt_at(PI_LITERAL, 8, buf[0], lane - 1, idx, bit);
					rc_put(lane, idx, bit);
				}
				rc_run(9);
				++uncomp_size;
			}
			is_initialized = 1;
			fast_restart(read_pos);
		}
		for (;;) {
			if (read_pos - read_ahead >= limit || rc_pending_reaches(XZB_LZMA2_CHUNK_MAX - XZB_LOOP_INPUT_MAX)) break;
			if (read_pos >= size) { if (read_ahead == 0) break; }
			if (mf_stalled) break;
			if constexpr (SM::RCQ != 0) { while (rq_head - S.rcq_tail > SM::RCQ - 128u) { } }   // ring space for one symbol
			uint32_t len, back;
			fast_pop(&back, &len);
			if (back == XZB_BACK_STALL) { mf_stalled = true; break; }
			encode_symbol(back, len, uncomp_size);
			uncomp_size += len;
		}
		rc_flush();
	}
};

// Fast mode (presets 0-3), warp 1: lzma_lzma_optimum_fast (lzma_encoder_optimum_fast.c:19-169) looks only at
// the match store, the window and the four reps -- never at probabilities or the range coder -- so the
// decisions can be taken ahead of the coding warp.  The reps are mirrored here with the update rules
// of encode_symbol (lzma_encoder.c:152-229).
template <class SM, class ENC>
__device__ inline void xzb_w_fast_parser_main(SM &S, ENC &P)
{
	uint32_t my_epoch = 0, k = 0;
	bool idle = true;
	for (;;) {
		const uint32_t e = S.f_epoch;
		if (e != my_epoch) {
			__threadfence_block();
			my_epoch = e; k = 0; idle = false;
			P.read_pos = S.f_start_pos; P.read_ahead = 0;
			P.rep0 = P.rep1 = P.rep2 = P.rep3 = 0;
		}
		if (S.m_exit) return;
		if (idle) { __nanosleep(200); continue; }
		if (P.read_pos >= P.size && P.read_ahead == 0) { idle = true; continue; }  // lzma_encoder.c:345-351: nothing left to decide
		if (k - S.f_consumed >= XZB_FRING) { __nanosleep(20); continue; }
		uint32_t back, len;
		P.optimum_fast(&back, &len);
		if (P.mf_stalled) { back = XZB_BACK_STALL; len = 1; idle = true; }
		const uint32_t slot = k % XZB_FRING;
		__syncwarp();
		if (P.lane == 0) {
			S.f_back[slot] = back; S.f_lenra[slot] = len | (P.read_ahead << 16); S.f_rpos[slot] = P.read_pos;
			asm volatile("" ::: "memory");   // one warp's shared-memory stores are performed in order
			S.f_tag[slot] = ((uint64_t)my_epoch << 32) | (uint64_t)(k + 1);
		}
		++k;
		P.read_ahead -= len;
		if (back < XZB_REPS) {  // rep_match :178-207 (a short rep leaves the reps alone)
			if (back == 1) { const uint32_t d = P.rep1; P.rep1 = P.rep0; P.rep0 = d; }
			else if (back == 2) { const uint32_t d = P.rep2; P.rep2 = P.rep1; P.rep1 = P.rep0; P.rep0 = d; }
			else if (back == 3) { const uint32_t d = P.rep3; P.rep3 = P.rep2; P.rep2 = P.rep1; P.rep1 = P.rep0; P.rep0 = d; }
		} else if (back != XZB_BACK_LITERAL && back != XZB_BACK_STALL) {  // match :152-175
			P.rep3 = P.rep2; P.rep2 = P.rep1; P.rep1 = P.rep0; P.rep0 = back - XZB_REPS;
		}
	}
}

// ------------------------------------------------------------------------------------------------
// Coder warp (kernels whose shared-memory struct has RCQ != 0): the low/range recurrence and the byte output of the
// range encoder (range_encoder.h:135-263).  The coding warp only adapts the probabilities and queues
// (probability before adaptation | bit << 12 | direct << 13) records, 0x8000 = flush the chunk; this warp turns them
// into the chunk's bytes and publishes rc_out_pos + rc_cache_size for the LZMA2 chunk-size test (rc_pending_reaches).
// ------------------------------------------------------------------------------------------------
template <class SM, class ENC>
__device__ inline void xzb_w_coder_main(SM &S, ENC &H)
{
	const uint32_t lane = H.lane;
	H.rc_low = 0; H.rc_cache_size = 1; H.rc_range = 0xFFFFFFFFu; H.rc_cache = 0; H.rc_out_pos = 0;
	uint32_t tail = 0, flushes = 0;
	bool fresh = true;
	for (;;) {
		uint32_t head;
		while ((head = S.rcq_head) == tail) { if (S.m_exit) return; }
		asm volatile("" ::: "memory");
		if (fresh) { H.rc_out = S.rcq_out; H.rc_out_pos = 0; fresh = false; }
		const uint32_t n = xzb_min(head - tail, 32u);
		const uint32_t w = lane < n ? (uint32_t)S.rcq[(tail + lane) & (SM::RCQ - 1)] : 0u;
		for (uint32_t i = 0; i < n; ++i) {
			const uint32_t wi = __shfl_sync(WFULL, w, i);
			if (wi & 0x8000u) {
				if (H.rc_range < (1u << 24)) { H.rc_shift_low(); H.rc_range <<= 8; }
				for (int k = 0; k < 5; ++k) H.rc_shift_low();
				const uint32_t sz = H.rc_out_pos;
				H.rc_low = 0; H.rc_cache_size = 1; H.rc_range = 0xFFFFFFFFu; H.rc_cache = 0; H.rc_out_pos = 0;
				++flushes;
				fresh = true;   // anything after a flush marker belongs to the next chunk; the coding warp waits for us first
				__syncwarp();
				if (lane == 0) {
					S.rcq_out_pos = sz;
					S.rcq_T = 1;
					S.rcq_tail = tail + i + 1;
					__threadfence_block();
					S.rcq_flushes = flushes;
				}
			} else if (wi & 0x2000u) {
				H.rc_step(0xFFFF, (wi >> 12) & 1);
			} else {
				H.rc_step_prob(wi & 0xFFF, (wi >> 12) & 1);
			}
		}
		tail += n;
		__syncwarp();
		if (lane == 0) {
			S.rcq_T = H.rc_out_pos + H.rc_cache_size;
			asm volatile("" ::: "memory");
			S.rcq_tail = tail;
		}
	}
}

// Shared memory of the fast-mode kernel xzb_k_parse_fast (presets 0-3): lzma_lzma_optimum_fast needs no price table
// and no opts[] array, so a Block's coder state is 38 KB.  CODER_WARP: the range coder's arithmetic runs on a warp
// of its own (xzb_w_coder_main), fed through rcq; otherwise the coding warp runs it and rcq stays unused.
template <bool CODER_WARP>
struct FS {
	static constexpr uint32_t RCQ_SIZE = 2048;
	static constexpr uint32_t RCQ = CODER_WARP ? RCQ_SIZE : 0u;
	static constexpr bool FAST = true;
	alignas(16) xzb_pair ring_mp[32][8];
	uint32_t ring_mh[32];
	uint32_t m_dist[XZB_MATCH_LEN_MAX + 1];
	uint16_t m_len[XZB_MATCH_LEN_MAX + 1], m_len2[XZB_MATCH_LEN_MAX + 1];
	uint8_t m_mb[XZB_MATCH_LEN_MAX + 1 + 2];
	xzb_prob probs[PI_TOTAL + 2];
	alignas(8) uint16_t rc_bits[72];
	volatile uint64_t f_tag[XZB_FRING];
	volatile uint32_t f_back[XZB_FRING], f_lenra[XZB_FRING], f_rpos[XZB_FRING];
	volatile uint32_t f_epoch, f_start_pos, f_consumed, m_exit;
	alignas(4) uint16_t rcq[RCQ_SIZE];
	uint8_t *rcq_out;
	volatile uint32_t rcq_head, rcq_tail, rcq_T, rcq_flushes, rcq_out_pos;
};

struct XzbEncJob;

// lzma2_encode over the whole block (lzma2_encoder.c:134-259), warp version of xzb_lzma2_encode_block
template <class ENC>
__device__ inline int xzb_w_lzma2_encode_block(ENC &E, const XzbParams &P, uint8_t *out, uint32_t out_cap, uint32_t *out_pos_ptr,
		uint32_t *n_chunks_lzma, uint32_t *n_chunks_raw)
{
	uint32_t out_pos = *out_pos_ptr;
	bool need_properties = true, need_state_reset = false, need_dictionary_reset = true;
	for (;;) {
		if (E.size - E.read_pos + E.read_ahead == 0) {
			if (out_pos >= out_cap) return XZB_BUF_ERROR;
			if (E.lane == 0) out[out_pos] = 0;
			++out_pos;
			break;
		}
		if (out_pos + XZB_LZMA2_HEADER_MAX + XZB_LZMA2_CHUNK_MAX > out_cap) return XZB_BUF_ERROR;
		if (need_state_reset) E.reset();
		const uint32_t hdr = need_properties ? 6u : 5u;
		const uint32_t limit = E.read_pos - E.read_ahead + XZB_LZMA2_UNCOMPRESSED_MAX - XZB_MATCH_LEN_MAX;
		const uint32_t read_start = E.read_pos - E.read_ahead;
		E.set_rc_out(out + out_pos + hdr);
		E.encode_chunk(limit);
		if (E.mf_stalled) return XZB_MF_STALL;
		const uint32_t compressed_size = E.rc_out_pos;
		uint32_t uncompressed_size = E.read_pos - E.read_ahead - read_start;
		__syncwarp();
		if (compressed_size >= uncompressed_size) {
			++*n_chunks_raw;
			uncompressed_size += E.read_ahead;
			E.read_ahead = 0;
			if constexpr (ENC::FAST) E.fast_restart(E.read_pos);
			if (E.lane == 0) {
				out[out_pos] = need_dictionary_reset ? 1 : 2;
				out[out_pos + 1] = (uint8_t)((uncompressed_size - 1) >> 8);
				out[out_pos + 2] = (uint8_t)((uncompressed_size - 1) & 0xFF);
			}
			out_pos += 3;
			need_dictionary_reset = false;
			need_state_reset = true;
			const uint8_t *src = E.buf + E.read_pos - uncompressed_size;
			for (uint32_t i = E.lane; i < uncompressed_size; i += 32) out[out_pos + i] = src[i];
			out_pos += uncompressed_size;
			__syncwarp();
			continue;
		}
		++*n_chunks_lzma;
		if (E.lane == 0) {
			uint8_t *h = out + out_pos;
			uint32_t pos = 0;
			uint8_t c;
			if (need_properties) c = need_dictionary_reset ? 0x80 + (3 << 5) : 0x80 + (2 << 5);
			else c = need_state_reset ? 0x80 + (1 << 5) : 0x80;
			uint32_t sz = uncompressed_size - 1;
			h[pos++] = (uint8_t)(c + (sz >> 16));
			h[pos++] = (uint8_t)((sz >> 8) & 0xFF);
			h[pos++] = (uint8_t)(sz & 0xFF);
			sz = compressed_size - 1;
			h[pos++] = (uint8_t)(sz >> 8);
			h[pos++] = (uint8_t)(sz & 0xFF);
			if (need_properties) h[pos++] = P.lclppb;
		}
		need_properties = false; need_state_reset = false; need_dictionary_reset = false;
		out_pos += hdr + compressed_size;
	}
	*out_pos_ptr = out_pos;
	return XZB_OK;
}
