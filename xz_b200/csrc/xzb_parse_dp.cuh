// xzb_parse_dp.cuh -- normal-mode parser (lzma_lzma_optimum_normal) as a dataflow DP: one chain
// warp carries the true recurrence, a team of worker warps does everything else (device only).
//
// Same decisions, bit for bit, as lzma_encoder_optimum_normal.c:270-858.  The reference walks the
// DP nodes one by one; for node `cur` it (1) reads the best way to reach cur, (2) derives state and
// reps, (3) prices the literal / short rep into cur+1 and (4) tries every rep and match candidate
// of cur against opts[cur+len].  Only (1)-(3) form a recurrence from node to node; (4) is the bulk of
// the work and is needed no earlier than `len` nodes later.  Hence:
//
//   * CHAIN WARP (warp 0): per node -- take the finished slot, derive state/reps from the source
//     node's record, price the literal, publish the node record {price, cur_and_1_price, state,
//     reps, match byte}, then finish slot cur+1: wait until every earlier node has pushed what can
//     land there, gather the workers' best candidates (one lane per worker ring, two redux.min), and
//     settle literal / short rep against them in registers.  It also runs helper1 (node 0),
//     backward(), the range coder and the LZMA2 chunker between segments.
//   * WORKER WARPS (W = 12, or 3 when nice_len > 127): worker w owns nodes w+1, w+1+W, ...
//     Before the node is reached it prepares the position's state-independent facts (match list,
//     get_dist_len_price of every length, the "match + literal + rep0" candidates minus two state
//     bits, the plain literal price).  When the chain warp publishes the node record it does the window
//     compares for the four reps and pushes the node's candidates into ITS OWN ring of 16-byte
//     slots (price, back, packed link incl. the target's match byte, back_2) -- private rings, so no
//     atomics -- in three waves ordered by distance (targets <= +3, <= +8, rest), publishing a phase
//     flag after each; the chain warp only waits for the wave it needs.  "Literal + rep0" needs the
//     chain's verdict on slot cur+1 and comes last; only the one slot it lands on waits for it.
//   * Exactness of ties (strict '<' keeps the first candidate in the reference's program order,
//     DESIGN.md F3): inside a ring candidates are applied class by class in program order; across
//     rings the gather prefers the lower source node; the one candidate that must be applied late
//     (literal + rep0 needs the outcome of slot cur+1) wins ties against its own node's later classes.
//
// lzma_encoder_optimum_normal.c line references are given per function.
#pragma once
#include "xzb_parse_warp.cuh"

// XZB_DP_PROF: cycle counters of the chain warp / worker 0 of block 0, printed at kernel end (development aid)
// Hand-offs between the warps of one CTA go through shared memory only.  Writer: data, DP_RELEASE(), flag.
// Reader: flag (volatile), DP_ACQUIRE(), data -- the loads are control-dependent on the flag, the barrier only
// keeps the compiler from hoisting them.  The writer needs no fence.cta either: a warp's shared-memory stores are
// performed in program order by the SM's in-order shared-memory pipeline, and a fence would wait for every store in
// flight (DESIGN.md section 8 lists the fence among the dead ends).
#define DP_RELEASE() asm volatile("" ::: "memory")
#define DP_ACQUIRE() asm volatile("" ::: "memory")
#ifdef XZB_DP_PROF
#define DP_T(v) const long long v = clock64()
#define DP_ACC(i, a, b) do { if (blockIdx.x == 0) S.prof[i] += (unsigned long long)((b) - (a)); } while (0)
#define DP_CNT(i) do { if (blockIdx.x == 0) S.prof[i] += 1; } while (0)
#define DP_CNTA(i) do { if (blockIdx.x == 0) atomicAdd(&S.prof[i], 1ull); } while (0)   // from any worker warp
#else
#define DP_T(v)
#define DP_ACC(i, a, b)
#define DP_CNT(i)
#define DP_CNTA(i)
#endif
#define DP_NPROF 62u

// 16-byte shared-memory records are handed over with ONE vector store and polled with ONE vector load (an aligned
// 16-byte access of one lane is a single shared-memory transaction, so the reader sees all of it or none)
__device__ __forceinline__ uint4 dp_lds128(const volatile void *p)
{
	uint4 v;
	asm volatile("ld.volatile.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"((uint32_t)__cvta_generic_to_shared(const_cast<const void *>(p))) : "memory");
	return v;
}
__device__ __forceinline__ uint2 dp_lds64(const volatile void *p)
{
	uint2 v;
	asm volatile("ld.volatile.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"((uint32_t)__cvta_generic_to_shared(const_cast<const void *>(p))) : "memory");
	return v;
}
__device__ __forceinline__ void dp_sts64(volatile void *p, const uint2 v)
{
	asm volatile("st.volatile.shared.v2.u32 [%0], {%1, %2};" :: "r"((uint32_t)__cvta_generic_to_shared(const_cast<void *>(p))), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ void dp_sts128(volatile void *p, const uint4 v)
{
	asm volatile("st.volatile.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"((uint32_t)__cvta_generic_to_shared(const_cast<void *>(p))), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// The owner of node c looks at slot c once node c - DP_PEEK_LAG is final.  With lag 1 the record is late for a large
// share of the nodes; with lag 2 it is not, and the candidate that leads the slot then is nearly always the final winner.
#define DP_PEEK_LAG 2u
#define DP_WMAX 12u
#define DP_POOL 3088u                 // ring slots: 12 workers x (256 + 1) or 3 workers x (1024 + 1); +1 skews the rings over the banks
#define DP_NR 1024u                   // node-record / phase-flag ring capacity (>= ring size)
#define DP_PLAIN_POOL 1536u           // per worker: [len - 2] = { get_dist_len_price | match byte << 16, dist }
#define DP_STALL_HDR 0xFFFFFFFFu
#define DP_NONE 0xFFFFFFFFu

// packed link of a slot / final node: d1 = target - pos_prev (1..273), flags bit0 prev_1_is_literal,
// bit1 prev_2, d2 = pos_prev - pos_prev_2 (x + literal: len_x + 1), mb = byte at target - rep0 - 1
#define DP_META(d1, flags, d2, mb) ((d1) | ((flags) << 9) | ((d2) << 11) | ((mb) << 20))
#define DP_D1(m) ((m) & 0x1FFu)
#define DP_FLAGS(m) (((m) >> 9) & 3u)
#define DP_D2(m) (((m) >> 11) & 0x1FFu)
#define DP_MB(m) (((m) >> 20) & 0xFFu)
// node the candidate starts from (reps / state come from there)
#define DP_SRC(target, m) ((target) - DP_D1(m) - (DP_FLAGS(m) == 0 ? 0u : (DP_FLAGS(m) == 1 ? 1u : DP_D2(m))))

// worker -> chain warp: state-independent facts of one block position, ONE 16-byte record written with a single
// 16-byte store and polled with a single 16-byte load:
//   x = tagn(node) + 1 (complete), y = hdr: count | longest << 16 (match store header), DP_STALL_HDR = watchdog,
//   z = buf[p] | buf[p-1] << 8, w = get_literal_price(..., match_mode = false, ...)
typedef uint4 DpPrep;

#define DP_RCQ 4096u                  // coded-bit ring to the coder warp (16-bit records); 4096: the coder warp keeps up with a batch (DESIGN.md section 8)
struct DS {  // dynamic shared memory of xzb_k_parse_dp
	static constexpr uint32_t RCQ = DP_RCQ;
	static constexpr bool FAST = false;
	// ---- coder state shared with WarpEncT's methods ----
	uint32_t len_prices[2][XZB_POS_STATES_MAX][XZB_LEN_SYMBOLS];
	uint32_t dist_slot_prices[XZB_DIST_STATES][XZB_DIST_SLOTS];
	uint32_t dist_prices[XZB_DIST_STATES][XZB_FULL_DISTANCES];
	uint32_t align_prices[XZB_ALIGN_SIZE];
	uint32_t len_counters[2][XZB_POS_STATES_MAX];
	alignas(16) xzb_pair ring_mp[32][8];
	uint32_t ring_mh[32];
	uint32_t m_dist[XZB_MATCH_LEN_MAX + 1];
	uint16_t m_len[XZB_MATCH_LEN_MAX + 1];
	xzb_prob probs[PI_TOTAL + 2];
	uint8_t prices[128];
	alignas(8) uint16_t rc_bits[72];
	// ---- DP ----
	alignas(16) uint4 ring_pool[DP_POOL];   // worker rings: x price, y back_prev, z DP_META, w back_prev_2; doubles as the symbol stack
	uint4 n_reps[DP_NR];                    // node records (ring): reps[]
	alignas(8) uint2 n_info[DP_NR];         //   x = price of the node, y = state | match byte buf[p - rep0 - 1] << 8
	uint32_t n_c1[DP_NR];                   //   cur_and_1_price
	uint32_t o_back[XZB_OPTS], o_meta[XZB_OPTS], o_back2[XZB_OPTS];   // final links, read by backward()
	alignas(16) uint4 pb[XZB_STATES][XZB_POS_STATES_MAX][2];  // price bundles, see build_bundles()
	alignas(16) DpPrep prep[32];
	alignas(8) uint2 plain_pool[DP_PLAIN_POOL];
	volatile uint32_t ph[DP_NR];            // (tagn(node) << 2) | waves of the node that are pushed (1..3)
	volatile uint32_t seg_epoch, seg_P0, seg_position0, fin_node, nil_node, seg_stop, m_exit;
	uint32_t len_end_sh;
	volatile uint32_t idle[DP_WMAX + 1];      // workers 0..W-1, [W] = the gather warp
	alignas(16) uint4 part[32];              // gather warp -> chain warp: the workers' best candidate of node t
	// owner worker -> chain warp: node t resolved ahead of time for the candidate that led slot t when the worker looked
	// (res_b = that candidate, res_a = the reps it implies, res_c = { is_match0 + literal price, short-rep bundle,
	// state, tagn(t) + 1 }); the chain warp uses it when that candidate is the one that finally wins the slot
	alignas(16) uint4 res_a[32], res_b[32], res_c[32];
	// chain warp -> coder warp: probability before adaptation | bit << 12 | direct << 13; 0x8000 = flush the chunk
	alignas(4) uint16_t rcq[DP_RCQ];
	uint8_t *rcq_out;                        // where the chunk's bytes go (set before the chunk's first bit)
	volatile uint32_t rcq_head, rcq_tail;    // bits pushed / consumed
	volatile uint32_t rcq_T;                 // rc_out_pos + rc_cache_size at rcq_tail
	volatile uint32_t rcq_flushes, rcq_out_pos;   // chunks finished, compressed size of the last one
	volatile uint32_t part_tag[32];          // tagn(t) + 1
	// owner worker -> gather / chain warp, per node c (ring c & 31): { tagn(c) + 1, the slot c's "literal + rep0" lands on
	// while its push is pending, else 0 }; written before the node's first phase flag with ONE 8-byte store.  Only nodes
	// t-2 .. t-W-1 are ever read, and node c-32's worker has finished it before slot c can finish, so 32 entries suffice.
	alignas(8) uint2 lr[32];
#ifdef XZB_DP_PROF
	unsigned long long prof[DP_NPROF];
#endif
};

struct DpEnc : WarpEncT<DS> {
	uint32_t W, rsize, rmask, rstride, plain_stride;   // team geometry (depends on nice_len)
	uint32_t epoch;                           // chain warp: current segment
	uint32_t sym_cur, sym_end;                // symbol stack [sym_cur, sym_end) left over from the last backward()
	uint32_t *trace; uint32_t trace_cap, trace_n;
#ifdef XZB_DP_PROF
	long long t_stop = 0;                     // chain warp: clock64() when the last segment was stopped
#endif

	__device__ DpEnc(DS &s, uint32_t l) : WarpEncT<DS>(s, l) {}

	__device__ void reset() { WarpEncT<DS>::reset(); sym_cur = sym_end = 0; }  // lzma_lzma_encoder_reset: opts_*_index = 0
	__device__ __forceinline__ uint2 *sym_stack() const { return reinterpret_cast<uint2 *>(&S.ring_pool[0]); }  // 4096 x {back, len}
	static __device__ __forceinline__ uint32_t st_lit(uint32_t s) { return s <= 3 ? 0 : (s <= 9 ? s - 3 : s - 6); }
	static __device__ __forceinline__ uint32_t tagn(uint32_t ep, uint32_t node) { return ((ep & 0x3FFFu) << 16) | node; }

	// Bit prices of the state-dependent flags, pre-added the way helper1/helper2 use them (:329-340, :520-548, :602-618):
	// [0] = { is_match 0, is_match 1 + is_rep 0 (normal match), is_match 1 + is_rep 1 (rep match), + short rep }
	// [1] = rep match + get_pure_rep_price(0..3)
	__device__ void build_bundles()
	{
		for (uint32_t t = lane; t < XZB_STATES * num_pos_states; t += 32) {
			const uint32_t st = t / num_pos_states, ps = t - st * num_pos_states;
			const uint32_t m0 = pr0(PI_IS_MATCH + (st << 4) + ps), m1 = pr1(PI_IS_MATCH + (st << 4) + ps);
			const uint32_t e0 = pr0(PI_IS_REP + st), e1 = pr1(PI_IS_REP + st);
			const uint32_t g0 = pr0(PI_IS_REP0 + st), g1 = pr1(PI_IS_REP0 + st);
			const uint32_t l0 = pr0(PI_IS_REP0_LONG + (st << 4) + ps), l1 = pr1(PI_IS_REP0_LONG + (st << 4) + ps);
			const uint32_t h0 = pr0(PI_IS_REP1 + st), h1 = pr1(PI_IS_REP1 + st);
			const uint32_t k0 = pr0(PI_IS_REP2 + st), k1 = pr1(PI_IS_REP2 + st);
			const uint32_t R = m1 + e1;
			S.pb[st][ps][0] = make_uint4(m0, m1 + e0, R, R + g0 + l0);
			S.pb[st][ps][1] = make_uint4(R + g0 + l1, R + g1 + h0, R + g1 + h1 + k0, R + g1 + h1 + k1);
		}
		__syncwarp();
	}
	static __device__ __forceinline__ uint32_t bundle_rep(const uint4 &b1, uint32_t r) { return r == 0 ? b1.x : r == 1 ? b1.y : r == 2 ? b1.z : b1.w; }

	// node reached through link (back, meta, back2) from a source node with state st_src and reps rs: its state and reps
	// (:453-497), branch-free
	static __device__ __forceinline__ void derive(const uint4 link, const uint32_t st_src, const uint4 rs, uint32_t &st, uint4 &r)
	{
		const uint32_t d1 = DP_D1(link.z), fl = DP_FLAGS(link.z);
		const uint32_t xb = fl == 3 ? link.w : link.y;   // the symbol that last changed the reps
		const bool step1 = fl == 0 && d1 == 1;           // literal or short rep from cur - 1
		const bool hi = st_src >= XZB_LIT_STATES;
		const bool is_new = xb >= XZB_REPS && xb != XZB_BACK_LITERAL;   // a match: new rep0, the others shift
		// literal (reps kept), short rep / rep0 (xb == 0: kept), rep xb (moved to the front), match
		r.x = is_new ? xb - XZB_REPS : (xb == 1 ? rs.y : xb == 2 ? rs.z : xb == 3 ? rs.w : rs.x);
		r.y = (is_new || xb == 1 || xb == 2 || xb == 3) ? rs.x : rs.y;
		r.z = (is_new || xb == 2 || xb == 3) ? rs.y : rs.z;
		r.w = (is_new || xb == 3) ? rs.z : rs.w;
		const uint32_t st_rm = is_new ? (hi ? 10u : 7u) : (hi ? 11u : 8u);   // plain match / rep from the source
		const uint32_t st_1 = xb == 0 ? (hi ? 11u : 9u) : st_lit(st_src);       // short rep / literal
		st = step1 ? st_1 : (fl != 0 ? 8u : st_rm);                            // "... + literal + rep0" ends in state 8
	}

	// one lane per candidate into ring `rg`; targets of the valid lanes are distinct (strict '<': an earlier candidate keeps the slot)
	__device__ __forceinline__ void push(uint4 *rg, bool valid, uint32_t target, uint32_t price, uint32_t back, uint32_t meta, uint32_t back2)
	{
		if (valid) {
			uint4 *s = &rg[target & rmask];
			if (price < s->x) *s = make_uint4(price, back, meta, back2);
		}
	}

	// ---- backward (:222-263): links -> symbol stack, first symbol returned ----
	__device__ void backward(uint32_t *len_res, uint32_t *back_res, uint32_t end)
	{
		__syncwarp();
		uint32_t k = XZB_OPTS;
		if (lane == 0) {
			// the walk only reads o_*; the stack overlays the rings, which the (finished) DP no longer needs
			uint2 *stk = sym_stack();
			uint32_t c = end;
			while (c != 0) {
				const uint32_t meta = S.o_meta[c], back = S.o_back[c];
				const uint32_t d1 = DP_D1(meta), fl = DP_FLAGS(meta);
				stk[--k] = make_uint2(back, d1);
				uint32_t pp = c - d1;
				if (fl & 1) {
					stk[--k] = make_uint2(XZB_BACK_LITERAL, 1);
					pp -= 1;
					if (fl & 2) {
						const uint32_t xl = DP_D2(meta) - 1;
						stk[--k] = make_uint2(S.o_back2[c], xl);
						pp -= xl;
					}
				}
				c = pp;
			}
		}
		k = __shfl_sync(WFULL, k, 0);
		__syncwarp();
		const uint2 first = sym_stack()[k];
		*back_res = first.x; *len_res = first.y;
		sym_cur = k + 1; sym_end = XZB_OPTS;
	}

	__device__ void rings_clear()
	{
		for (uint32_t i = lane; i < W * rstride; i += 32) S.ring_pool[i] = make_uint4(XZB_INFINITY_PRICE, 0, 0, 0);
		__syncwarp();
	}

	// ---- helper1 (:270-439): node 0 of a segment, pushed into ring 0 while the workers are idle.
	// Returns len_end or 0xFFFFFFFF when the symbol is decided. ----
	__device__ uint32_t helper1(uint32_t *back_res, uint32_t *len_res, uint32_t position)
	{
		uint32_t len_main, mcount;
		if (read_ahead == 0) {
			len_main = mf_find(&mcount);
		} else {
			len_main = longest_match_length;
			mcount = matches_count;
		}
		if (mf_stalled) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return 0xFFFFFFFFu; }
		const uint32_t buf_avail = xzb_min(mf_avail() + 1, XZB_MATCH_LEN_MAX);
		if (buf_avail < 2) { *back_res = XZB_BACK_LITERAL; *len_res = 1; return 0xFFFFFFFFu; }
		const uint32_t p0 = read_pos - 1;
		const uint8_t *b = buf + p0;
		uint32_t rl[4];
		rep_lens4(b, buf_avail, rl);
		uint32_t rep_max_index = 0;
		for (uint32_t i = 1; i < XZB_REPS; ++i) if (rl[i] > rl[rep_max_index]) rep_max_index = i;
		if (rl[rep_max_index] >= nice_len) {
			*back_res = rep_max_index; *len_res = rl[rep_max_index];
			mf_skip(*len_res - 1); return 0xFFFFFFFFu;
		}
		if (len_main >= nice_len) {
			*back_res = S.m_dist[mcount - 1] + XZB_REPS; *len_res = len_main;
			mf_skip(len_main - 1); return 0xFFFFFFFFu;
		}
		const uint32_t current_byte = b[0];
		const uint32_t match_byte = *(b - rep0 - 1);
		if (len_main < 2 && current_byte != match_byte && rl[rep_max_index] < 2) {
			*back_res = XZB_BACK_LITERAL; *len_res = 1; return 0xFFFFFFFFu;
		}
		build_bundles();   // probabilities are frozen from here to the end of the segment
		const uint32_t pos_state = position & pos_mask;
		const uint4 b0 = S.pb[state][pos_state][0], b1 = S.pb[state][pos_state][1];
		const uint32_t lit = literal_price(position, b[-1], state >= XZB_LIT_STATES, match_byte, current_byte);
		uint32_t price1 = b0.x + lit;
		uint32_t back1 = XZB_BACK_LITERAL;
		if (match_byte == current_byte) {
			const uint32_t srp = b0.w;
			if (srp < price1) { price1 = srp; back1 = 0; }
		}
		const uint32_t len_end = xzb_max(len_main, rl[rep_max_index]);
		if (len_end < 2) { *back_res = back1; *len_res = 1; return 0xFFFFFFFFu; }
		rings_clear();
		uint4 *rg = &S.ring_pool[0];
		if (lane == 0) {
			S.n_info[0] = make_uint2(0u, state);
			S.n_reps[0] = make_uint4(rep0, rep1, rep2, rep3);
			rg[1] = make_uint4(price1, back1, DP_META(1u, 0u, 0u, (uint32_t)*(b + 1 - rep0 - 1)), 0);
		}
		__syncwarp();
		for (uint32_t i = 0; i < XZB_REPS; ++i) {
			const uint32_t rep_len = rl[i];
			if (rep_len < 2) continue;
			const uint32_t price = bundle_rep(b1, i);
			const uint32_t rr = rep_of(i);
			for (uint32_t l = 2 + lane; l - lane <= rep_len; l += 32) {
				const bool v = l <= rep_len;
				uint32_t p = 0, mbt = 0;
				if (v) { p = price + len_price(1, l, pos_state); mbt = *(b + l - rr - 1); }
				push(rg, v, l, p, i, DP_META(l, 0u, 0u, mbt), 0);
			}
			__syncwarp();
		}
		const uint32_t start = rl[0] >= 2 ? rl[0] + 1 : 2;
		if (start <= len_main) {
			for (uint32_t l = start + lane; l - lane <= len_main; l += 32) {
				const bool v = l <= len_main;
				uint32_t p = 0, dist = 0, mbt = 0;
				if (v) {
					const uint32_t i = match_index_for(l, mcount);
					dist = S.m_dist[i];
					p = b0.y + dist_len_price(dist, l, pos_state);
					mbt = *(b + l - dist - 1);
				}
				push(rg, v, l, p, dist + XZB_REPS, DP_META(l, 0u, 0u, mbt), 0);
			}
			__syncwarp();
		}
		return len_end;
	}

	// ---- chain warp: the workers' best candidate for node t (every ring's slot t; lower source node wins ties) ----
	__device__ __forceinline__ uint4 gather(uint32_t t)
	{
		uint4 v = make_uint4(XZB_INFINITY_PRICE, 0, 0, 0);
		uint4 *e = &S.ring_pool[(lane < W ? lane : 0) * rstride + (t & rmask)];
		if (lane < W) { v = *e; e->x = XZB_INFINITY_PRICE; }   // the slot is free for node t + rsize
		return best_of(t, v);
	}
	// the best of the lanes' ring entries for node t (lanes >= W hold none)
	__device__ __forceinline__ uint4 best_of(uint32_t t, uint4 v)
	{
		const uint32_t m = __reduce_min_sync(WFULL, v.x);
		const uint32_t src = (lane < W && v.x == m) ? DP_SRC(t, v.z) : DP_NONE;
		const uint32_t s = __reduce_min_sync(WFULL, src);
		const uint32_t win = (uint32_t)__ffs((int)__ballot_sync(WFULL, src == s)) - 1;
		v.x = m;
		v.y = __shfl_sync(WFULL, v.y, win); v.z = __shfl_sync(WFULL, v.z, win); v.w = __shfl_sync(WFULL, v.w, win);
		return v;
	}
	__device__ __forceinline__ bool ph_ok(uint32_t node, uint32_t need) const
	{
		const uint32_t v = S.ph[node & rmask];
		return (v >> 2) == tagn(epoch, node) && (v & 3) >= need;
	}
	// the slot node's "literal + rep0" is still to be pushed onto, else 0.  Loaded right behind the node's phase flag:
	// loads are performed in order, so once the flag is seen the record is the one written before it (a node without a
	// record -- fewer than 2 bytes left -- has no such candidate).
	__device__ __forceinline__ uint32_t lr_target(uint32_t node) const
	{
		const uint2 r = dp_lds64(&S.lr[node & 31]);
		return r.x == tagn(epoch, node) + 1 ? r.y : 0u;
	}
	// Every candidate that can land on node t has been pushed: nodes t-2 .. t-W-1 are checked -- the wave that covers t,
	// and no "literal + rep0" pending onto t (node t-1 only reaches t through the chain warp's registers; anything older
	// shares its worker with a checked node that has already started, and a worker finishes a node, "literal + rep0"
	// included, before it starts the next).
	// Lane d - 2 also loads slot t of ring wr, the ring of node t - d, with every poll, behind that node's flag and record:
	// when the last flag is seen, v already is the final entry (no further round trip), and the slot is cleared for node
	// t + rsize.  Returns false when the segment was stopped meanwhile.
	__device__ __forceinline__ bool wait_deadlines(uint32_t t, uint32_t wr, uint4 &v)
	{
		const uint32_t d = lane + 2;
		uint4 *const e = &S.ring_pool[(lane < W ? wr : 0) * rstride + (t & rmask)];
		const bool mine = d <= W + 1 && t > d;   // node t - d >= 1
		const uint32_t need = d <= 3 ? 1u : (d <= 8 ? 2u : 3u);
#ifdef XZB_DP_PROF
		const uint32_t dbin = d <= 4 ? d - 2 : d <= 8 ? 3 : 4;
		uint32_t miss = 0;   // what this lane still waited for at the last failed poll: 1 = the phase flag, 2 = "literal + rep0"
#endif
		for (uint32_t it = 0;; ++it) {
			const bool okp = !mine || ph_ok(t - d, need);
			const uint32_t lt = mine ? lr_target(t - d) : 0u;
			if (lane < W) v = dp_lds128(e);
			const bool ok = okp && lt != t;
			if (__all_sync(WFULL, ok)) break;
#ifdef XZB_DP_PROF
			if (it == 0 && !ok && blockIdx.x == 0) atomicAdd(&S.prof[24 + dbin], 1ull);   // which node the slot waits for
			miss = ok ? 0u : (okp ? 2u : 1u);
#endif
			if ((it & 15) == 15 && (S.seg_stop != DP_NONE || S.m_exit)) return false;
		}
#ifdef XZB_DP_PROF
		if (miss != 0) DP_CNTA(44 + 5 * (miss - 1) + dbin);
#endif
		DP_ACQUIRE();
		if (lane < W) e->x = XZB_INFINITY_PRICE;
		else v = make_uint4(XZB_INFINITY_PRICE, 0, 0, 0);
		return true;
	}
	__device__ __forceinline__ void wait_all_complete(uint32_t cur)   // nodes 1 .. cur-1 have pushed everything
	{
		const uint32_t d = lane + 1;
		const bool mine = d <= W && cur > d;
		for (;;) {
			const bool okp = !mine || ph_ok(cur - d, 3);
			const uint32_t lt = mine ? lr_target(cur - d) : 0u;
			const bool ok = okp && lt == 0;
			if (__all_sync(WFULL, ok)) break;
		}
		DP_ACQUIRE();
	}

	// ---- lzma_lzma_optimum_normal (:802-858); helper2's (:442-799) chain part ----
	__device__ void optimum_normal(uint32_t *back_res, uint32_t *len_res, uint32_t position)
	{
		if (sym_cur != sym_end) {
			const uint2 s = sym_stack()[sym_cur++];
			*back_res = s.x; *len_res = s.y;
			return;
		}
		if (read_ahead == 0) {
			if (match_price_count >= (1 << 7)) fill_dist_prices();
			if (align_price_count >= XZB_ALIGN_SIZE) fill_align_prices();
		}
		DP_T(h0);
		uint32_t le = helper1(back_res, len_res, position);   // len_end as far as this warp knows
		{ DP_T(h1); if (lane == 0) DP_ACC(16, h0, h1); }
		if (le == 0xFFFFFFFFu) return;
		// node c sits at block position P0 + c, LZMA position position + c
		const uint32_t P0 = read_pos - 1;
		epoch = (epoch + 1) & 0x3FFF;
		if (epoch == 0) epoch = 1;
		__syncwarp();
		if (lane == 0) {
			S.len_end_sh = le;
			S.seg_P0 = P0; S.seg_position0 = position; S.seg_stop = DP_NONE;
			S.fin_node = tagn(epoch, 0); S.nil_node = tagn(epoch, 0) << 1;
			__threadfence_block();
			S.seg_epoch = epoch;
		}
		__syncwarp();
		uint4 Wn = gather(1);   // node 1: literal / short rep of helper1

		uint32_t cur;
		uint4 Rn = dp_lds128(&S.prep[1]);   // the prep record of the next node is requested one node early; its tag is checked on use
#ifdef XZB_DP_PROF
		long long t_prev = clock64();
#endif
		for (cur = 1;; ++cur) {
			// ---- for (cur = 1; cur < len_end; ++cur): len_end grows with the workers' pushes ----
			if (cur >= le) {
				le = *(volatile uint32_t *)&S.len_end_sh;
				if (cur >= le) {
					DP_T(s0);
					wait_all_complete(cur);
					DP_T(s1);
					if (lane == 0) { DP_ACC(5, s0, s1); DP_CNT(6); }
					le = *(volatile uint32_t *)&S.len_end_sh;
					if (cur >= le) break;
				}
			}
			DP_T(t0);
#ifdef XZB_DP_PROF
			if (lane == 0) DP_ACC(7, t_prev, t0);   // loop top: from the end of the previous node's body
#endif
			// ---- the owner's facts about this position (mf_find equivalent): one 16-byte poll ----
			uint4 R = Rn;
			{
				const uint32_t want = tagn(epoch, cur) + 1;
				const uint4 *rp = &S.prep[cur & 31];
				while (R.x != want) R = dp_lds128(rp);
				DP_ACQUIRE();
				Rn = dp_lds128(&S.prep[(cur + 1) & 31]);
			}
			DP_T(t1);
			const uint32_t hdr = R.y;
			if (hdr == DP_STALL_HDR) { mf_stalled = true; break; }
			const uint32_t longest = hdr >> 16;
			matches_count = hdr & 0xFFFF; longest_match_length = longest;
			if (longest >= nice_len) {  // :846-847; the next call's helper1 wants the match list itself
				mf_find(&matches_count);
				break;
			}
			++read_pos; ++read_ahead;
			const uint32_t p = P0 + cur;
			const uint32_t pos = position + cur;
			const uint32_t ps = pos & pos_mask;
			const uint32_t baf = xzb_min(size - p, XZB_OPTS - 1 - cur);   // buf_avail_full
			const uint32_t cb = R.z & 0xFF;

			// ---- node cur: link -> state, reps (:453-497); taken from the owner's look-ahead when it resolved this very link ----
			const uint32_t meta = Wn.z;
			const uint4 Qc = dp_lds128(&S.res_c[cur & 31]);   // the tag first: the data is at least as new
			const uint4 Qb = dp_lds128(&S.res_b[cur & 31]);
			const uint4 Qa = dp_lds128(&S.res_a[cur & 31]);
			// A 16-byte shared-memory load of a whole warp is served in quarter-warp phases, so while the owner is writing the
			// record the lanes can see different versions: the vote makes the decision uniform (a lane that passed the test
			// has a complete, matching record of its own -- tag loaded first).
			const bool hit = __all_sync(WFULL, Qc.w == tagn(epoch, cur) + 1 && Qb.x == Wn.x && Qb.y == Wn.y && Qb.z == Wn.z && Qb.w == Wn.w);
			uint32_t st, r0, r1, r2, r3;
			if (hit) {
				st = Qc.z; r0 = Qa.x; r1 = Qa.y; r2 = Qa.z; r3 = Qa.w;
				if (lane == 0) DP_CNT(20);
			} else {
#ifdef XZB_DP_PROF
				if (lane == 0) {
					if (DP_FLAGS(meta) == 0 && DP_D1(meta) == 1) DP_CNT(23);      // literal / short rep won: nothing to look ahead at
					else if (Qc.w != tagn(epoch, cur) + 1) DP_CNT(22);             // record not there (yet)
					else DP_CNT(21);                                               // another candidate won
				}
#endif
				const uint32_t src = DP_SRC(cur, meta);
				const uint32_t st_src = S.n_info[src & rmask].y & 0xFF;
				const uint4 rs = S.n_reps[src & rmask];
				uint4 r;
				derive(Wn, st_src, rs, st, r);
				r0 = r.x; r1 = r.y; r2 = r.z; r3 = r.w;
			}
			const uint32_t mb = DP_MB(meta);           // = buf[p - r0 - 1]
			const uint32_t cur_price = Wn.x;
			{
				// every lane stores the same values (no divergent block on the chain)
				const uint32_t k = cur & rmask;
				S.n_info[k] = make_uint2(cur_price, st | (mb << 8));
				S.n_reps[k] = make_uint4(r0, r1, r2, r3);
				S.o_back[cur] = Wn.y; S.o_meta[cur] = meta; S.o_back2[cur] = Wn.w;
				DP_RELEASE();
				*(volatile uint32_t *)&S.fin_node = tagn(epoch, cur);   // the owner of node cur may push now (n_c1 follows with nil_node)
			}
#ifdef XZB_DP_PROF
			if (cur == 1 && t_stop != 0) { DP_T(f1); if (lane == 0) { DP_ACC(33, t_stop, f1); DP_CNT(34); } }   // seg_stop -> next first fin_node
#endif
			// first look at the gather warp's record for slot cur + 1 (usually there already; the loads overlap the pricing below)
			const uint32_t wantp = tagn(epoch, cur + 1) + 1;
			const volatile uint32_t *tp = &S.part_tag[(cur + 1) & 31];
			const uint4 *dp = &S.part[(cur + 1) & 31];
			uint32_t tg = *tp;
			uint4 N = dp_lds128(dp);
			// ---- literal and short rep (:499-548), in registers ----
			uint32_t c1, srp;
			if (hit) {
				c1 = cur_price + Qc.x; srp = cur_price + Qc.y;
			} else {
				const uint4 b0 = S.pb[st][ps][0];
				const uint32_t lit = st < XZB_LIT_STATES ? R.w : literal_price(pos, R.z >> 8, true, mb, cb);
				c1 = cur_price + b0.x + lit;      // cur_and_1_price
				srp = cur_price + b0.w;
			}
			const uint32_t mb1 = baf >= 2 ? (uint32_t)*(buf + p - r0) : 0u;   // match byte of cur + 1 if it is reached by literal / short rep
			// ---- finish slot cur + 1 ----
			DP_T(t2);
			while (tg != wantp) { tg = *tp; N = dp_lds128(dp); }   // loads issue in order: the data is at least as new as its tag
			DP_ACQUIRE();
			DP_T(t3);
			bool next_is_literal = false;
			if (c1 < N.x) { N = make_uint4(c1, XZB_BACK_LITERAL, DP_META(1u, 0u, 0u, mb1), 0); next_is_literal = true; }
			if (mb == cb && !(DP_D1(N.z) > 1 && N.y == 0)) {
				if (srp <= N.x) { N = make_uint4(srp, 0, DP_META(1u, 0u, 0u, mb1), 0); next_is_literal = true; }
			}
			S.n_c1[cur & rmask] = c1;
			DP_RELEASE();
			*(volatile uint32_t *)&S.nil_node = (tagn(epoch, cur) << 1) | (next_is_literal ? 1u : 0u);   // releases the owner's "literal + rep0"
			Wn = N;
			DP_T(t4);
			if (lane == 0) { DP_ACC(0, t0, t1); DP_ACC(1, t1, t2); DP_ACC(2, t2, t3); DP_ACC(3, t3, t4); DP_CNT(4); }
#ifdef XZB_DP_PROF
			t_prev = clock64();
#endif
		}
		// stop the team, then the end node's link (its slot is final: every earlier node has pushed what can reach it)
		__syncwarp();
		if (lane == 0) { S.o_back[cur] = Wn.y; S.o_meta[cur] = Wn.z; S.o_back2[cur] = Wn.w; __threadfence_block(); S.seg_stop = cur; }
		DP_T(i0);
#ifdef XZB_DP_PROF
		t_stop = i0;
#endif
		for (;;) {
			const bool ok = lane > W || S.idle[lane] == epoch;
			if (__all_sync(WFULL, ok)) break;
		}
		DP_ACQUIRE();
		DP_T(i1);
		backward(len_res, back_res, cur);
		{ DP_T(i2); if (lane == 0) { DP_ACC(17, i0, i1); DP_ACC(18, i1, i2); DP_CNT(19); } }
	}

	// the i-th (len, dist) pair of block position p straight from the match store
	__device__ __forceinline__ xzb_pair match_pair(uint32_t p, uint32_t count, uint32_t i) const
	{
		const xzb_pair *inl = g_mp + (size_t)p * 8;
		if (count <= 8 || i < 7) {
			const uint2 v = *reinterpret_cast<const uint2 *>(inl + i);
			return xzb_pair{ v.x, v.y };
		}
		const uint2 v = __ldcg(reinterpret_cast<const uint2 *>(g_ovf + inl[7].len + (i - 7)));
		return xzb_pair{ v.x, v.y };
	}

	// State-independent part of the "match + literal + rep0" candidate of one match (:729-790), one lane per match.
	// pk = len | len_test_2 << 9 | (byte at target - dist - 1) << 18; rel = its price minus (normal_match_price +
	// is_match[state_after_match] bit 0).
	__device__ __forceinline__ void mlr_eval(uint32_t p, uint32_t pos, uint32_t ps, const xzb_pair pr, uint32_t &pk, uint32_t &dist, uint32_t &rel) const
	{
		const uint8_t *b = buf + p;
		const uint32_t L = XZB_PAIR_LEN(pr.len), r = XZB_PAIR_LEN2(pr.len), mbm = XZB_PAIR_MB(pr.len);
		dist = pr.dist;
		const uint32_t avail1 = size - p;
		const uint32_t limit = xzb_min(avail1, L + 1 + nice_len);
		uint32_t lt2 = 0, mbt = 0;
		rel = 0;
		if (L + 1 < limit) lt2 = xzb_min(L + 1 + r, limit) - (L + 1);
		if (lt2 >= 2) {
			const uint32_t psn2 = (pos + L + 1) & pos_mask;
			rel = dist_len_price(dist, L, ps) + literal_price_matched_lane(pos + L, b[L - 1], mbm, b[L])
					+ S.pb[4][psn2][1].x + len_price(1, lt2, psn2);
			mbt = *(b + L + 1 + lt2 - dist - 1);
		} else {
			lt2 = 0;
		}
		pk = L | (lt2 << 9) | (mbt << 18);
	}

	__device__ __forceinline__ uint32_t sym_nbits(uint32_t back, uint32_t len, uint32_t ps) const
	{
		if (back == XZB_BACK_LITERAL) return 9;
		const bool m = back >= XZB_REPS;
		const uint32_t pre_n = m ? 2u : (back <= 1 ? 4u : 5u);
		if (!m && len == 1) return pre_n;   // short rep
		return LenDist(pre_n, m ? 0u : 1u, ps, len, m ? back - XZB_REPS : 0xFFFFFFFFu).n;
	}

	// ---- the run backward() just stacked, coded as one batch ----
	// Codes the symbols from sym_cur - 1 (the one optimum_normal returned) on, with exactly encode_symbol's records and
	// side effects, up to the first symbol before which one of encode_chunk's limit tests might hold: the uncompressed
	// one is exact from the lengths; the compressed one takes the bound of rc_pending_reaches, read once, plus the
	// records of the batch's earlier symbols (each record the coder warp takes meanwhile lowers the queue by one and
	// raises its count by at most one).  The symbols from there on are left on the stack for the exact per-symbol loop.
	//   32 symbols at a time, lane j = symbol j: lengths and record counts by warp scans, state and reps by a uniform
	//   loop, the length-price counters per (coder, pos_state) group; each lane writes its symbol's records to a staging
	//   area.  Then the records go out 32 at a time in coding order: equal probability indices of a window hand the value
	//   on in lane order, and a window stops at the first record of a symbol whose length prices are refreshed
	//   (length_count: the refresh sees every earlier symbol's adaptations and none of its own, DESIGN.md F2).
	__device__ void encode_batch(uint32_t limit)
	{
		const uint32_t s0 = sym_cur - 1, n = sym_end - s0;
		uint32_t cb0 = 0;
		if (lane == 0) { const uint32_t tail = S.rcq_tail; asm volatile("" ::: "memory"); cb0 = S.rcq_T + (rq_head - tail) + 4; }
		cb0 = __shfl_sync(WFULL, cb0, 0);
		const uint32_t p0 = read_pos - read_ahead, lt = (1u << lane) - 1;
		uint32_t *const len_ctr = &S.len_counters[0][0];   // [which * XZB_POS_STATES_MAX + pos_state]
		// the records of 32 symbols (at most 48 each) are staged behind the symbol stack, in the workers' idle rings
		static_assert((DP_POOL - XZB_OPTS / 2) * sizeof(uint4) >= 32 * 48 * sizeof(uint16_t), "batch staging");
		uint16_t *const stg = reinterpret_cast<uint16_t *>(&S.ring_pool[XZB_OPTS / 2]);
		uint32_t done = 0, off = 0, nrec = 0;   // symbols, bytes and records of the batch so far
		bool cut = false;
		while (done < n && !cut) {
			const bool in = done + lane < n;
			const uint2 sy = in ? sym_stack()[s0 + done + lane] : make_uint2(0u, 0u);
			const uint32_t back = sy.x, len = sy.y;
			const uint32_t pos = uncomp_size + off;   // + the lengths before this lane's symbol
			uint32_t lx = len;
#pragma unroll
			for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(WFULL, lx, d); if (lane >= d) lx += o; }
			lx -= len;
			const uint32_t ps = (pos + lx) & pos_mask;
			const uint32_t nb = in ? sym_nbits(back, len, ps) : 0u;
			uint32_t bx = nb;
#pragma unroll
			for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(WFULL, bx, d); if (lane >= d) bx += o; }
			bx -= nb;
			const bool stop = in && done + lane != 0 && (p0 + off + lx >= limit || cb0 + nrec + bx >= XZB_LZMA2_CHUNK_MAX - XZB_LOOP_INPUT_MAX);
			const uint32_t sm = __ballot_sync(WFULL, stop);
			const uint32_t nw = sm ? (uint32_t)__ffs((int)sm) - 1 : xzb_min(n - done, 32u);
			cut = sm != 0;
			if (nw == 0) break;
			const bool v = lane < nw;
			// state and reps before each symbol (encode_symbol's updates); they end before the first symbol not coded
			uint32_t st = 0, r0 = 0;
			for (uint32_t u = 0; u < nw; ++u) {
				const uint32_t b = __shfl_sync(WFULL, back, u), l = __shfl_sync(WFULL, len, u);
				if (lane == u) { st = state; r0 = rep0; }
				const bool hi = state >= XZB_LIT_STATES;
				if (b == XZB_BACK_LITERAL) {
					state = hi ? (state <= 9 ? state - 3 : state - 6) : (state <= 3 ? 0 : state - 3);
				} else if (b >= XZB_REPS) {
					state = hi ? 10 : 7;
					rep3 = rep2; rep2 = rep1; rep1 = rep0; rep0 = b - XZB_REPS;
				} else {
					if (b != 0) {
						const uint32_t d = b == 1 ? rep1 : b == 2 ? rep2 : rep3;
						if (b == 3) rep3 = rep2;
						if (b >= 2) rep2 = rep1;
						rep1 = rep0; rep0 = d;
					}
					state = l == 1 ? (hi ? 11 : 9) : (hi ? 11 : 8);
				}
			}
			const bool lit = back == XZB_BACK_LITERAL, is_m = !lit && back >= XZB_REPS;
			n_symbols += nw;
			match_price_count += __popc(__ballot_sync(WFULL, v && is_m));
			align_price_count += __popc(__ballot_sync(WFULL, v && is_m && xzb_dist_slot(back - XZB_REPS) >= XZB_DIST_MODEL_END));
			// length_count of every length in the window: k-th decrement of a counter that starts at c0, refreshed at 0
			const bool has_len = v && !lit && (is_m || len != 1);
			const uint32_t ci = (is_m ? 0u : XZB_POS_STATES_MAX) + ps;
			const uint32_t grp = __match_any_sync(WFULL, has_len ? ci : 0x100u + lane);
			const uint32_t c0 = has_len ? len_ctr[ci] : 1u, L = len_table_size;
			const uint32_t kd = __popc(grp & lt) + 1;
			const bool refresh = has_len && kd >= c0 && (kd - c0) % L == 0;
			__syncwarp();
			if (has_len && (grp >> lane) == 1) {
				const uint32_t K = __popc(grp);
				len_ctr[ci] = K < c0 ? c0 - K : L - (K - c0) % L;
			}
			if (trace != nullptr && v && trace_n + lane < trace_cap) { const uint32_t t = 3 * (trace_n + lane); trace[t] = pos + lx; trace[t + 1] = back; trace[t + 2] = len; }
			trace_n += nw;
			// every lane writes its symbol's records (idx | bit << 14 | direct << 15) in encode_symbol's order
			if (v) {
				uint16_t *const o = stg + bx;
				const uint32_t ism = PI_IS_MATCH + (st << 4) + ps;
				if (lit) {   // encode_literal
					const uint32_t p = p0 + off + lx, cb = buf[p];
					const uint32_t mb = st >= XZB_LIT_STATES ? buf[p - r0 - 1] : 0u;
					const uint32_t sub = PI_LITERAL + 3u * (((((pos + lx) << 8) + buf[p - 1]) & literal_mask) << lc);
					o[0] = (uint16_t)ism;
#pragma unroll
					for (uint32_t j = 0; j < 8; ++j) {
						const uint32_t pre = (cb | 0x100) >> (8 - j), bit = (cb >> (7 - j)) & 1;
						uint32_t idx = sub + pre;
						if (st >= XZB_LIT_STATES) {
							const uint32_t mo = ((cb ^ mb) >> (8 - j)) == 0 ? 0x100u : 0u;
							idx += mo + (((mb >> (7 - j)) & 1) ? mo : 0u);
						}
						o[1 + j] = (uint16_t)(idx | (bit << 14));
					}
				} else {     // the prefix of encode_symbol's match / rep match, then encode_len_dist
					const uint32_t pre_n = is_m ? 2u : (back <= 1 ? 4u : 5u);
					o[0] = (uint16_t)(ism | (1u << 14));
					o[1] = (uint16_t)((PI_IS_REP + st) | (is_m ? 0u : 1u << 14));
					if (!is_m) {
						o[2] = (uint16_t)((PI_IS_REP0 + st) | (back != 0 ? 1u << 14 : 0u));
						o[3] = (uint16_t)(back == 0 ? (PI_IS_REP0_LONG + ism - PI_IS_MATCH) | (len != 1 ? 1u << 14 : 0u) : (PI_IS_REP1 + st) | (back != 1 ? 1u << 14 : 0u));
						if (back >= 2) o[4] = (uint16_t)((PI_IS_REP2 + st) | ((back - 2) << 14));
					}
					if (nb > pre_n) {
						const LenDist d(pre_n, is_m ? 0u : 1u, ps, len, is_m ? back - XZB_REPS : 0xFFFFFFFFu);
						for (uint32_t k = pre_n; k < nb; ++k) {
							uint32_t idx = 0, bit = 0;
							const bool dr = d.at(k, idx, bit);
							o[k] = (uint16_t)(idx | (bit << 14) | (dr ? 1u << 15 : 0u));
						}
					}
				}
			}
			__syncwarp();
			// then 32 records at a time, in coding order
			const uint32_t last = nw - 1;
			const uint32_t total = __shfl_sync(WFULL, bx + nb, last);
			uint32_t rmask = __ballot_sync(WFULL, refresh);
			uint32_t next = rmask ? __shfl_sync(WFULL, bx, __ffs((int)rmask) - 1) : total;   // first record of the next refresh symbol
			for (uint32_t r = 0;;) {
				while (rmask && next == r) {   // the refresh comes before that symbol's records
					const uint32_t j = (uint32_t)__ffs((int)rmask) - 1;
					rmask &= rmask - 1;
					length_update_prices(__shfl_sync(WFULL, is_m ? 0u : 1u, j), __shfl_sync(WFULL, ps, j));
					next = rmask ? __shfl_sync(WFULL, bx, __ffs((int)rmask) - 1) : total;
					if (lane == 0) DP_CNT(41);
				}
				if (r >= total) break;
				const uint32_t e = xzb_min(r + 32, next);
				const bool live = r + lane < e;
				const uint32_t w = live ? stg[r + lane] : 0x8000u;
				const bool direct = (w & 0x8000u) != 0;
				const uint32_t idx = w & 0x3FFFu, bit = (w >> 14) & 1;
				// equal indices: the value before adaptation is handed on in coding (= lane) order
				const uint32_t g = __match_any_sync(WFULL, direct ? 0x10000u + lane : idx);
				uint32_t pv = direct ? 0u : S.probs[idx];
				const uint32_t below = g & lt, rank = __popc(below);
				const uint32_t pred = below ? 31u - __clz(below) : lane;
				const uint32_t maxr = __reduce_max_sync(WFULL, rank);
				for (uint32_t t = 1; t <= maxr; ++t) {
					const uint32_t a = __shfl_sync(WFULL, bit ? pv - (pv >> 5) : pv + ((2048 - pv) >> 5), pred);
					if (rank == t) pv = a;
				}
				if (!direct && (g >> lane) == 1) S.probs[idx] = (xzb_prob)(bit ? pv - (pv >> 5) : pv + ((2048 - pv) >> 5));
#ifdef XZB_DP_PROF
				if (rq_head + 32u - S.rcq_tail > DP_RCQ) {
					DP_T(q0);
					while (rq_head + 32u - S.rcq_tail > DP_RCQ) { }
					DP_T(q1);
					if (lane == 0) DP_ACC(38, q0, q1);
				}
#endif
				while (rq_head + 32u - S.rcq_tail > DP_RCQ) { }   // ring space for the window
				if (live) S.rcq[(rq_head + lane) & (DP_RCQ - 1)] = (uint16_t)(direct ? 0x2000u | (bit << 12) : pv | (bit << 12));
				rc_run(e - r);
				r = e;
			}
			if (lane == 0) DP_ACC(37, 0, total);
			const uint32_t wl = __shfl_sync(WFULL, lx + len, last);
			off += wl; nrec += total; done += nw;
		}
		read_ahead -= off;
		uncomp_size += off;
		sym_cur = s0 + done;
		if (cut && lane == 0) DP_CNT(39);
	}

	// ---- lzma_lzma_encode for one LZMA2 chunk (lzma_encoder.c:266-436) ----
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
		}
		for (;;) {
			DP_T(l0);
			if (read_pos - read_ahead >= limit || rc_pending_reaches(XZB_LZMA2_CHUNK_MAX - XZB_LOOP_INPUT_MAX)) break;
			if (read_pos >= size) { if (read_ahead == 0) break; }
			if (mf_stalled) break;
#ifdef XZB_DP_PROF
			if (rq_head - S.rcq_tail > DP_RCQ - 128u) {
				DP_T(q0);
				while (rq_head - S.rcq_tail > DP_RCQ - 128u) { }
				DP_T(q1);
				if (lane == 0) { DP_ACC(31, q0, q1); DP_CNT(32); }
			}
#endif
			while (rq_head - S.rcq_tail > DP_RCQ - 128u) { }   // ring space for one symbol
			uint32_t len, back;
			const bool fresh = sym_cur == sym_end;   // no symbols stacked: optimum_normal decides, maybe by a DP
			DP_T(e0);
			optimum_normal(&back, &len, uncomp_size);
			DP_T(e1);
			if (mf_stalled) break;
			if (fresh && sym_cur != sym_end) {   // a DP stacked a run behind this symbol
#ifdef XZB_DP_PROF
				const uint32_t n0 = n_symbols;
#endif
				encode_batch(limit);
#ifdef XZB_DP_PROF
				DP_T(e2);
				if (lane == 0 && blockIdx.x == 0) { DP_ACC(42, l0, e0); DP_ACC(13, e0, e1); DP_ACC(35, e1, e2); DP_CNT(36); S.prof[15] += n_symbols - n0; }
#endif
				continue;
			}
#ifdef XZB_DP_PROF
			if (!fresh && lane == 0) DP_CNT(40);   // a stacked symbol left over by a cut batch
#endif
			if (trace != nullptr && lane == 0 && trace_n < trace_cap) { trace[3 * trace_n] = uncomp_size; trace[3 * trace_n + 1] = back; trace[3 * trace_n + 2] = len; }
			++trace_n;
			encode_symbol(back, len, uncomp_size);
			{ DP_T(e2); if (lane == 0) { DP_ACC(42, l0, e0); DP_ACC(13, e0, e1); DP_ACC(14, e1, e2); DP_CNT(15); DP_CNT(43); } }
			uncomp_size += len;
		}
		rc_flush();
	}
};

// ------------------------------------------------------------------------------------------------
// Coder warp: the low/range recurrence and the byte output of the range encoder (range_encoder.h:135-263).
// The chain warp only adapts the probabilities (which is all the DP's prices ever see) and queues
// (probability before adaptation, bit) records; this warp turns them into the chunk's bytes.
// ------------------------------------------------------------------------------------------------
__device__ inline void xzb_dp_coder_main(DS &S, DpEnc &H) { xzb_w_coder_main(S, H); }   // the generic form in xzb_parse_warp.cuh

// ------------------------------------------------------------------------------------------------
// Gather warp: for t = 2, 3, ... wait until every worker candidate for node t is pushed, reduce the
// workers' rings to the best one (DpEnc::gather) and hand it to the chain warp.  It runs as far
// ahead of the chain warp as the workers' phase flags allow.
// ------------------------------------------------------------------------------------------------
__device__ inline void xzb_dp_gather_main(DS &S, DpEnc &H)
{
	const uint32_t lane = H.lane;
	uint32_t my_epoch = 0;
	for (;;) {
		uint32_t e;
		while ((e = S.seg_epoch) == my_epoch) { if (S.m_exit) return; __nanosleep(100); }
		__threadfence_block();
		my_epoch = e;
		H.epoch = e;
		uint32_t wr = lane < H.W ? H.W - 1 - lane : 0u;   // ring of node t - (lane + 2): worker (t - lane - 3) mod W
		for (uint32_t t = 2; t < XZB_OPTS; ++t, wr = wr + 1 == H.W ? 0u : wr + 1) {
			uint4 v;
			if (!H.wait_deadlines(t, wr, v)) break;
			// slot (t & 31) is free: the chain warp consumed node t - 32 long ago (it cannot be more than W + 1 nodes behind)
			v = H.best_of(t, v);
			__syncwarp();
			if (lane == 0) {
				S.part[t & 31] = v;
				DP_RELEASE();
				S.part_tag[t & 31] = DpEnc::tagn(my_epoch, t) + 1;
			}
		}
		while (S.seg_stop == DP_NONE && S.seg_epoch == my_epoch && !S.m_exit) __nanosleep(50);
		__syncwarp(); __threadfence_block();
		if (lane == 0) S.idle[H.W] = my_epoch;
	}
}

// ------------------------------------------------------------------------------------------------
// Worker warp w: owns nodes w+1, w+1+W, ... of every segment (helper2 :550-796, the candidate part).
// ------------------------------------------------------------------------------------------------
struct DpNodeCands {   // one node's candidates, one lane each, as prepared by the owner
	// plain lengths: lane <-> length lane + 2
	bool v_r0, v_m;                        // rep0 of that length exists / a match candidate of that length exists
	uint32_t pr_r0, me_r0, pr_m, me_m, bk_m;
	// "match + literal + rep0": lane <-> match index
	bool v_c; uint32_t off_c, pr_c, me_c, bk2_c;
	// "rep0 + literal + rep0" (uniform)
	bool v_x0; uint32_t off_x0, pr_x0, me_x0;
};

__device__ inline void xzb_dp_worker_main(DS &S, DpEnc &H, const uint32_t w)
{
	const uint32_t lane = H.lane;
	const uint32_t W = H.W, rmask = H.rmask;
	uint4 *const rg = &S.ring_pool[w * H.rstride];
	uint2 *const PL = &S.plain_pool[w * H.plain_stride];
	uint32_t my_epoch = 0;
	for (;;) {
		uint32_t e;
		while ((e = S.seg_epoch) == my_epoch) { if (S.m_exit) return; __nanosleep(100); }
		__threadfence_block();
		my_epoch = e;
		const uint32_t P0 = S.seg_P0, position0 = S.seg_position0;
		for (uint32_t c = 1 + w; c < XZB_OPTS; c += W) {
			if (S.seg_stop != DP_NONE || S.m_exit) break;
			const uint32_t p = P0 + c;
			if (p >= H.size) break;
			const uint32_t pos = position0 + c;
			const uint32_t ps = pos & H.pos_mask;
			DP_T(wp);
			// =============== the position's state-independent facts ===============
			if (p + 1 > H.mf_done) {
				H.mf_wait(xzb_min(p + 64, H.size));
				if (H.mf_stalled) {
					if (lane == 0) dp_sts128(&S.prep[c & 31], make_uint4(DpEnc::tagn(my_epoch, c) + 1, DP_STALL_HDR, 0u, 0u));
					break;
				}
			}
			const uint32_t h = H.g_mh[p];
			const uint32_t count = h & 0xFFFF, longest = h >> 16;
			const uint8_t *b = H.buf + p;
			const uint32_t cb = b[0], pbyte = b[-1];
			uint32_t mL = 0, mdist = 0, mlt2 = 0, mrel = 0, mmbt = 0;   // match `lane`
			uint32_t lit_plain = 0;
			if (longest < H.nice_len) {
				lit_plain = H.literal_price(pos, pbyte, false, 0, cb);
				if (lane < count) {
					uint32_t pk;
					H.mlr_eval(p, pos, ps, H.match_pair(p, count, lane), pk, mdist, mrel);
					mL = pk & 0x1FF; mlt2 = (pk >> 9) & 0x1FF; mmbt = pk >> 18;
				}
				// per-length table: dist of the first match that covers the length
				const uint32_t c32 = xzb_min(count, 32u);
				for (uint32_t l = 2 + lane; l - lane <= longest; l += 32) {  // uniform trip count: shuffles inside
					uint32_t idx = 0;
					for (uint32_t j = 0; j + 1 < c32; ++j) { const uint32_t Lj = __shfl_sync(WFULL, mL, j); if (Lj < l) idx = j + 1; }
					uint32_t di = __shfl_sync(WFULL, mdist, idx & 31);
					if (count > 32 && idx == 31) {  // beyond the 32 lanes: walk the rest of the list
						for (uint32_t j = 31; j < count; ++j) {
							const xzb_pair pr = H.match_pair(p, count, j);
							di = pr.dist;
							if (XZB_PAIR_LEN(pr.len) >= l) break;
						}
					}
					if (l <= longest) {
						const uint32_t mbt = *(b + l - di - 1);
						PL[l - 2] = make_uint2(H.dist_len_price(di, l, ps) | (mbt << 16), di);
					}
				}
			}
			__syncwarp();   // the plain-length table of this position is written
			if (lane == 0) dp_sts128(&S.prep[c & 31], make_uint4(DpEnc::tagn(my_epoch, c) + 1, h, cb | (pbyte << 8), lit_plain));
			if (longest >= H.nice_len) break;  // the DP stops at this position
			const uint32_t want = DpEnc::tagn(my_epoch, c);
			bool gone = false;
			// =============== look ahead: resolve the node for the candidate that leads its slot now ===============
			// Once node c - DP_PEEK_LAG is final, almost everything that can reach slot c has been pushed.  The owner takes the
			// gather warp's result if it is out already, otherwise the best entry of the rings (read only), and works out what
			// the chain warp would otherwise derive on its critical path: state, reps, is_match0 + literal price, short-rep
			// bundle.  The chain warp uses the record only if that very candidate wins the slot in the end.
			bool have_p = false;              // window compare done ahead for the predicted reps rp_*
			uint32_t rmaskb_p = 0, cvw_p = 0, rp_0 = 0, rp_1 = 0, rp_2 = 0, rp_3 = 0;
			if (c >= 3) {
				// (every decision in these polling loops is lane 0's, broadcast: lanes that reach a loop at different times must
				// not leave it on different values of a flag that changes meanwhile -- the collectives below need the whole warp)
				uint32_t fnode = 0;
				__syncwarp();
				for (uint32_t it = 0;; ++it) {
					const uint32_t f = __shfl_sync(WFULL, S.fin_node, 0);
					fnode = f & 0xFFFF;
					if ((f >> 16) == (want >> 16) && fnode + DP_PEEK_LAG >= c) break;
					if ((it & 31) == 31 && __shfl_sync(WFULL, (uint32_t)(S.seg_stop != DP_NONE || S.seg_epoch != my_epoch || S.m_exit), 0)) { gone = true; break; }
				}
				if (gone) break;
				if (fnode < c) {
					uint4 v = make_uint4(XZB_INFINITY_PRICE, 0, 0, 0);
					const uint32_t ptag = __shfl_sync(WFULL, S.part_tag[c & 31], 0);
					if (ptag == want + 1) {
						v = dp_lds128(&S.part[c & 31]);
					} else {
						if (lane < W) v = dp_lds128(&S.ring_pool[lane * H.rstride + (c & rmask)]);
						const uint32_t m = __reduce_min_sync(WFULL, v.x);
						const uint32_t srcv = (lane < W && v.x == m) ? DP_SRC(c, v.z) : DP_NONE;
						const uint32_t s0 = __reduce_min_sync(WFULL, srcv);
						const uint32_t win = (uint32_t)__ffs((int)__ballot_sync(WFULL, srcv == s0)) - 1;
						v.x = m;
						v.y = __shfl_sync(WFULL, v.y, win); v.z = __shfl_sync(WFULL, v.z, win); v.w = __shfl_sync(WFULL, v.w, win);
					}
					if (v.x < XZB_INFINITY_PRICE) {
						const uint32_t src = DP_SRC(c, v.z);
						const uint32_t st_src = S.n_info[src & rmask].y & 0xFF;
						const uint4 rs = S.n_reps[src & rmask];
						uint32_t st_p; uint4 r_p;
						DpEnc::derive(v, st_src, rs, st_p, r_p);
						const uint4 b0p = S.pb[st_p][ps][0];
						const uint32_t lit_p = H.literal_price(pos, pbyte, true, DP_MB(v.z), cb);   // a rep or match leads here: matched literal
						if (lane == 0) {
							dp_sts128(&S.res_a[c & 31], r_p);
							dp_sts128(&S.res_b[c & 31], v);
							dp_sts128(&S.res_c[c & 31], make_uint4(b0p.x + lit_p, b0p.w, st_p, want + 1));
						}
						// the rep phase's round of window loads (below) for these reps, while the node is not final yet:
						// if the candidate wins, the loads are off the path from "node final" to "near candidates pushed"
						{
							const uint32_t bafp = xzb_min(H.size - p, XZB_OPTS - 1 - c);
							const uint32_t bav = xzb_min(bafp, H.nice_len);
							const uint32_t j = lane & 7, ri = lane >> 3;
							const uint32_t rq = ri == 0 ? r_p.x : ri == 1 ? r_p.y : ri == 2 ? r_p.z : r_p.w;
							const bool in = j < bav;
							const uint32_t av = in ? b[j] : 0u;
							cvw_p = in ? (b - rq - 1)[j] : 0x100u;
							rmaskb_p = __ballot_sync(WFULL, av != cvw_p);
							rp_0 = r_p.x; rp_1 = r_p.y; rp_2 = r_p.z; rp_3 = r_p.w;
							have_p = bafp >= 2;
						}
					}
				}
			}
			// =============== wait for the node itself ===============
			const uint32_t k = c & rmask;
			// Between here and the near-wave push nothing writes slots c + 2 and c + 3 of the own ring: this worker's earlier
			// nodes are done ("literal + rep0" included), and the gather warp clears a slot only when it reads it, which waits for this node's wave 1.
			// So the prices they hold now are the ones the push compares with, read off the path that follows the flag.
			const uint32_t near_old = lane < 2 ? rg[(c + 2 + lane) & rmask].x : 0u;
			DP_T(w0);
			__syncwarp();
			// The node record is loaded with every poll, after the flag: loads are performed in order, so when the flag says
			// the node is final, the record loaded after it is the final one -- one shared-memory round trip less after the flag.
			uint2 ni; uint4 rr;
			for (uint32_t it = 0;; ++it) {
				const uint32_t f = __shfl_sync(WFULL, S.fin_node, 0);
				ni = dp_lds64(&S.n_info[k]); rr = dp_lds128(&S.n_reps[k]);
				if ((f >> 16) == (want >> 16) && (f & 0xFFFF) >= c) break;
				if ((it & 31) == 31 && __shfl_sync(WFULL, (uint32_t)(S.seg_stop != DP_NONE || S.seg_epoch != my_epoch || S.m_exit), 0)) { gone = true; break; }
			}
			if (gone) break;
			DP_T(w1);
			DP_ACQUIRE();
			const uint32_t price = ni.x, st = ni.y & 0xFF, mb = ni.y >> 8;
			const uint32_t hr[4] = { rr.x, rr.y, rr.z, rr.w };
			const uint32_t baf = xzb_min(H.size - p, XZB_OPTS - 1 - c);   // buf_avail_full
			const uint32_t nice_len = H.nice_len, pos_mask = H.pos_mask;
			uint32_t lr_len = 0;   // "literal + rep0": len_test, 0 when there is no such candidate
			if (baf >= 2) {
				const uint32_t buf_avail = xzb_min(baf, nice_len);
				const uint4 b0 = S.pb[st][ps][0], b1 = S.pb[st][ps][1];
				// ---- one round of window loads for the rep phase: lane = (rep index, byte 0..7) ----
				uint32_t rmaskb, cvw;   // cvw: lane (r, j) holds buf[p - rep_r - 1 + j]
				if (have_p && hr[0] == rp_0 && hr[1] == rp_1 && hr[2] == rp_2 && hr[3] == rp_3) {
					rmaskb = rmaskb_p; cvw = cvw_p;   // done ahead by the look-ahead above
				} else {
					const uint32_t j = lane & 7;
					const uint32_t rq = hr[lane >> 3];
					const bool in = j < buf_avail;
					const uint32_t av = in ? b[j] : 0u;
					cvw = in ? (b - rq - 1)[j] : 0x100u;
					rmaskb = __ballot_sync(WFULL, av != cvw);
				}
				const uint32_t new_len = xzb_min(longest, buf_avail);   // :692-700 (the shortened last match has no X+literal+rep0 candidate)
				const uint32_t mg0 = rmaskb & 0xFF;
				const uint8_t *bb0 = b - hr[0] - 1;
				// Targets c + 2 and c + 3 are wanted first (the chain warp is about to finish them).  Whether rep0 / a match
				// of length 2 or 3 is a candidate follows from the compare mask alone: rep0 covers length L iff its first L
				// bytes match, and a match candidate of length L exists iff rep0 does not cover L (start_len, :690-715).
				bool near_done = false;
				{
					const bool other_reps = ((rmaskb >> 8) & 3) == 0 || ((rmaskb >> 16) & 3) == 0 || ((rmaskb >> 24) & 3) == 0;
					if (!other_reps && nice_len >= 8 && count <= 32) {
						const uint32_t L2 = lane + 2;
						const bool eqL = lane == 0 ? (mg0 & 3) == 0 : (mg0 & 7) == 0;
						const bool vr = lane < 2 && eqL, vmn = lane < 2 && !eqL && L2 <= new_len;
						const uint32_t lb = xzb_max((mg0 & 3) == 0 ? 2u : 0u, new_len >= 2 ? new_len : 0u);
						uint32_t prn = 0, men = 0, bkn = 0;
						const uint32_t nmb = __shfl_sync(WFULL, cvw, L2 & 7);   // rep0's bytes 0..7 sit in lanes 0..7
						if (vr) { prn = price + b1.x + H.len_price(1, L2, ps); men = DP_META(L2, 0u, 0u, L2 < buf_avail ? nmb : (uint32_t)bb0[L2]); }
						if (vmn) { const uint2 e2 = PL[L2 - 2]; prn = price + b0.y + (e2.x & 0xFFFF); men = DP_META(L2, 0u, 0u, e2.x >> 16); bkn = e2.y + XZB_REPS; }
						if ((vr || vmn) && prn < near_old) rg[(c + L2) & rmask] = make_uint4(prn, bkn, men, 0u);   // H.push against near_old
						__syncwarp();
						near_done = true;
						// "literal + rep0" of length exactly 2 (byte 0 differs, bytes 1-2 match, byte 3 does not) lands on c + 3:
						// its record goes out with wave 1; any other target is announced below, before wave 2
						if ((mg0 & 0xF) == 0x9 && lane == 0) dp_sts64(&S.lr[c & 31], make_uint2(want + 1, c + 3));
						DP_RELEASE();
						if (lane == 0) S.ph[k] = (want << 2) | 1u;
						// len_end only has to grow before this node's last phase flag (the chain warp waits for every node to be
						// complete before it ends the segment on len_end), so the atomic comes after the flag the gather waits for
						if (lane == 0 && lb) atomicMax(&S.len_end_sh, c + lb);
						{ DP_T(wn); if (lane == 0 && w == 0) { DP_ACC(29, w1, wn); DP_CNT(30); } }
					}
				}
				// "literal + rep0" (:562-597) exists iff rep0 misses byte 0 and matches bytes 1 .. len_test, len_test >= 2; it
				// lands on c + 1 + len_test.  Only whether it is pushed waits for the chain warp's verdict on slot c + 1, so
				// its target is announced before the phase flag of the wave that covers it (the near wave's own record
				// above) and the gather warp holds only that one slot for it.
				if (mg0 & 1) {
					const uint32_t lt = H.mlen_from(mg0, 1, buf_avail, b, bb0, xzb_min(baf, nice_len + 1)) - 1;
					if (lt >= 2) lr_len = lt;
				}
				if (lane == 0) dp_sts64(&S.lr[c & 31], make_uint2(want + 1, lr_len ? c + 1 + lr_len : 0u));
				uint32_t rlen[4];
#pragma unroll
				for (uint32_t ri = 0; ri < XZB_REPS; ++ri) {
					const uint32_t mg = (rmaskb >> (8 * ri)) & 0xFF;
					rlen[ri] = (mg & 3) ? 0u : H.mlen_from(mg, 2, buf_avail, b, b - hr[ri] - 1, buf_avail);
				}
				const uint32_t start_len = rlen[0] >= 2 ? rlen[0] + 1 : 2;
				const bool has_m = new_len >= start_len;
				const bool rare = (rlen[1] | rlen[2] | rlen[3]) >= 2 || xzb_max(rlen[0], new_len) > 33 || count > 32;
				uint32_t maxT = c + xzb_max(rlen[0], xzb_max(rlen[1], xzb_max(rlen[2], rlen[3])));
				if (has_m) maxT = xzb_max(maxT, c + new_len);

				if (lane == 0) atomicMax(&S.len_end_sh, maxT);
#ifdef XZB_DP_PROF
				if (lane == 0) {
					DP_CNTA(rare ? (near_done ? 57 : 58) : (near_done ? 54 : 55));
					if (lr_len == 2) DP_CNTA(56);   // lands on c + 3
					if (lr_len != 0) DP_CNTA(59);
				}
#endif

				// ---- this node's candidates, one lane each; the plain lengths first (the nearest targets are the urgent ones) ----
				DpNodeCands K;
				const uint32_t Ln = lane + 2;
				K.v_r0 = Ln <= rlen[0];
				K.v_m = has_m && Ln >= start_len && Ln <= new_len;
				K.pr_r0 = K.me_r0 = K.pr_m = K.me_m = K.bk_m = 0;
				{
					const uint32_t near_mb = __shfl_sync(WFULL, cvw, Ln & 7);   // rep0's bytes 0..7 sit in lanes 0..7
					if (K.v_r0) {
						const uint32_t mbt = (Ln < 8 && Ln < buf_avail) ? near_mb : (uint32_t)bb0[Ln];
						K.pr_r0 = price + b1.x + H.len_price(1, Ln, ps); K.me_r0 = DP_META(Ln, 0u, 0u, mbt);
					}
				}
				if (K.v_m) { const uint2 e2 = PL[Ln - 2]; K.pr_m = price + b0.y + (e2.x & 0xFFFF); K.me_m = DP_META(Ln, 0u, 0u, e2.x >> 16); K.bk_m = e2.y + XZB_REPS; }
				K.v_c = false; K.off_c = K.pr_c = K.me_c = K.bk2_c = 0;
				K.v_x0 = false; K.off_x0 = K.pr_x0 = K.me_x0 = 0;
				// the far classes ("match + literal + rep0" :729-790, "rep0 + literal + rep0" :635-687) land at c + 5 or later
				auto far_classes = [&]() {
					if (has_m && lane < count && mL >= start_len && mlt2 >= 2) {
						uint32_t lt2 = mlt2, rel = mrel, mbt = mmbt;
						if (baf < mL + 1 + lt2) {   // the DP window (or the block) ends inside the rep0 part: shorter rep0
							const uint32_t n2 = baf > mL + 1 ? baf - (mL + 1) : 0;
							if (n2 >= 2) {
								const uint32_t psn = (pos + mL + 1) & pos_mask;
								rel = rel - H.len_price(1, lt2, psn) + H.len_price(1, n2, psn);
								mbt = *(b + mL + 1 + n2 - mdist - 1);
							}
							lt2 = n2;
						}
						if (lt2 >= 2) {
							K.v_c = true;
							K.pr_c = price + b0.y + rel + S.pb[st < XZB_LIT_STATES ? 7u : 10u][(pos + mL) & pos_mask][0].x;
							K.off_c = c + mL + 1 + lt2;
							K.me_c = DP_META(lt2, 3u, mL + 1, mbt);
							K.bk2_c = mdist + XZB_REPS;
						}
					}
					uint32_t mt = __reduce_max_sync(WFULL, K.v_c ? K.off_c : 0u);
					if (rlen[0] >= 2) {
						const uint32_t len_test = rlen[0];
						uint32_t lt2 = len_test + 1;
						const uint32_t limit = xzb_min(baf, lt2 + nice_len);
						if (lt2 < limit) lt2 = H.mlen_from(rmaskb & 0xFF, lt2, buf_avail, b, bb0, limit);
						lt2 -= len_test + 1;
						if (lt2 >= 2) {
							const uint32_t st_x = st < XZB_LIT_STATES ? 8u : 11u;
							uint32_t psn = (pos + len_test) & pos_mask;
							const uint32_t calp = price + b1.x + H.len_price(1, len_test, ps) + S.pb[st_x][psn][0].x
									+ H.literal_price(pos + len_test, b[len_test - 1], true, bb0[len_test], b[len_test]);
							psn = (pos + len_test + 1) & pos_mask;
							K.v_x0 = true;
							K.pr_x0 = calp + S.pb[DpEnc::st_lit(st_x)][psn][1].x + H.len_price(1, lt2, psn);
							K.off_x0 = c + len_test + 1 + lt2;
							K.me_x0 = DP_META(lt2, 3u, len_test + 1, (uint32_t)bb0[len_test + 1 + lt2]);
							mt = xzb_max(mt, K.off_x0);
						}
					}
					if (lane == 0 && mt > maxT) atomicMax(&S.len_end_sh, mt);
				};

				// One wave: the classes in the reference's program order, restricted to targets in (c + lo, c + hi].
				auto wave = [&](const uint32_t lo, const uint32_t hi) {
					const bool inL = Ln > lo && Ln <= hi;
					H.push(rg, K.v_r0 && inL, c + Ln, K.pr_r0, 0, K.me_r0, 0);
					__syncwarp();
					if (K.v_x0 && K.off_x0 > c + lo && K.off_x0 <= c + hi) { H.push(rg, lane == 0, K.off_x0, K.pr_x0, 0, K.me_x0, 0); __syncwarp(); }
					const bool vc = K.v_c && K.off_c > c + lo && K.off_c <= c + hi;
					const uint32_t vm = __ballot_sync(WFULL, vc);
					if (vm) {
						const uint32_t same = __match_any_sync(WFULL, vc ? K.off_c : DP_NONE - lane);
						const bool clash = __any_sync(WFULL, vc && (same & (same - 1)) != 0);
						if (!clash) {
							H.push(rg, vc, K.off_c, K.pr_c, 0, K.me_c, K.bk2_c);
							__syncwarp();
						} else {
							uint32_t todo = vm;
							while (todo) {   // two candidates want the same slot: one at a time, in match order
								const uint32_t j = (uint32_t)__ffs((int)todo) - 1;
								todo &= todo - 1;
								H.push(rg, lane == j, K.off_c, K.pr_c, 0, K.me_c, K.bk2_c);
								__syncwarp();
							}
						}
					}
					H.push(rg, K.v_m && inL, c + Ln, K.pr_m, K.bk_m, K.me_m, 0);
					__syncwarp();
				};
				if (!rare) {
					if (!near_done) {                     // only plain lengths 2 and 3 can land here
						wave(0, 3);
						__syncwarp(); DP_RELEASE();
						if (lane == 0) S.ph[k] = (want << 2) | 1u;
					}
					far_classes();
					{ DP_T(w2); if (lane == 0 && w == 0) { DP_ACC(8, w0, w1); DP_ACC(9, w1, w2); DP_CNT(10); } }
					wave(3, 8);
					__syncwarp(); DP_RELEASE();
					if (lane == 0) S.ph[k] = (want << 2) | 2u;
					wave(8, 0xFFFFu);
				} else {
					// uncommon shapes (a second rep matches, very long candidates, > 32 matches): everything in the
					// reference's order in one go
					far_classes();
#pragma unroll
					for (uint32_t ri = 0; ri < XZB_REPS; ++ri) {
						const uint32_t len_test = rlen[ri];
						if (len_test < 2) continue;
						const uint8_t *bb = b - hr[ri] - 1;
						const uint32_t prc = price + DpEnc::bundle_rep(b1, ri);
						for (uint32_t l = 2 + lane; l - lane <= len_test; l += 32) {
							const bool v = l <= len_test && !(near_done && l <= 3);   // slots c+2 / c+3 are already pushed and may be consumed
							uint32_t pp = 0, mbt = 0;
							if (v) { pp = prc + H.len_price(1, l, ps); mbt = bb[l]; }
							H.push(rg, v, c + l, pp, ri, DP_META(l, 0u, 0u, mbt), 0);
						}
						__syncwarp();
						if (ri == 0) {
							if (K.v_x0) { H.push(rg, lane == 0, K.off_x0, K.pr_x0, 0, K.me_x0, 0); __syncwarp(); }
							continue;
						}
						uint32_t lt2 = len_test + 1;
						const uint32_t limit = xzb_min(baf, lt2 + nice_len);
						const uint32_t mg = (rmaskb >> (8 * ri)) & 0xFF;
						if (lt2 < limit) lt2 = H.mlen_from(mg, lt2, buf_avail, b, bb, limit);
						lt2 -= len_test + 1;
						if (lt2 >= 2) {
							const uint32_t st_x = st < XZB_LIT_STATES ? 8u : 11u;
							uint32_t psn = (pos + len_test) & pos_mask;
							const uint32_t calp = prc + H.len_price(1, len_test, ps) + S.pb[st_x][psn][0].x
									+ H.literal_price(pos + len_test, b[len_test - 1], true, bb[len_test], b[len_test]);
							psn = (pos + len_test + 1) & pos_mask;
							const uint32_t pp = calp + S.pb[DpEnc::st_lit(st_x)][psn][1].x + H.len_price(1, lt2, psn);
							const uint32_t offset = c + len_test + 1 + lt2;
							if (lane == 0) atomicMax(&S.len_end_sh, offset);
							H.push(rg, lane == 0, offset, pp, 0, DP_META(lt2, 3u, len_test + 1, (uint32_t)bb[len_test + 1 + lt2]), ri);
							__syncwarp();
						}
					}
					if (has_m) {
						const uint32_t nmp = price + b0.y;
						const uint32_t s2 = st < XZB_LIT_STATES ? 7u : 10u;
						for (uint32_t base = 0; base < count; base += 32) {
							const uint32_t i = base + lane;
							uint32_t off = 0, pp = 0, L = 0, dist = 0, lt2 = 0, mbt = 0;
							bool valid = false;
							if (i < count) {
								uint32_t rel;
								if (base == 0) { L = mL; lt2 = mlt2; mbt = mmbt; dist = mdist; rel = mrel; }
								else { uint32_t pk; H.mlr_eval(p, pos, ps, H.match_pair(p, count, i), pk, dist, rel); L = pk & 0x1FF; lt2 = (pk >> 9) & 0x1FF; mbt = pk >> 18; }
								if (L >= start_len && lt2 >= 2) {
									if (baf < L + 1 + lt2) {
										const uint32_t n2 = baf > L + 1 ? baf - (L + 1) : 0;
										if (n2 >= 2) {
											const uint32_t psn = (pos + L + 1) & pos_mask;
											rel = rel - H.len_price(1, lt2, psn) + H.len_price(1, n2, psn);
											mbt = *(b + L + 1 + n2 - dist - 1);
										}
										lt2 = n2;
									}
									if (lt2 >= 2) {
										valid = true;
										pp = nmp + rel + S.pb[s2][(pos + L) & pos_mask][0].x;
										off = c + L + 1 + lt2;
									}
								}
							}
							const uint32_t mx = __reduce_max_sync(WFULL, valid ? off : 0u);
							if (lane == 0 && mx) atomicMax(&S.len_end_sh, mx);
							uint32_t todo = __ballot_sync(WFULL, valid);
							while (todo) {   // in match order
								const uint32_t j = (uint32_t)__ffs((int)todo) - 1;
								todo &= todo - 1;
								H.push(rg, lane == j, off, pp, 0, DP_META(lt2, 3u, L + 1, mbt), dist + XZB_REPS);
								__syncwarp();
							}
						}
						for (uint32_t l = start_len + lane; l - lane <= new_len; l += 32) {
							const bool v = l <= new_len && !(near_done && l <= 3);
							uint32_t pp = 0, dist = 0, mbt = 0;
							if (v) { const uint2 e2 = PL[l - 2]; pp = nmp + (e2.x & 0xFFFF); mbt = e2.x >> 16; dist = e2.y; }
							H.push(rg, v, c + l, pp, dist + XZB_REPS, DP_META(l, 0u, 0u, mbt), 0);
						}
						__syncwarp();
					}
				}
			}
			__syncwarp(); DP_RELEASE();
			if (lane == 0) S.ph[k] = (want << 2) | 3u;
			{ DP_T(w3); if (lane == 0 && w == 0) { DP_ACC(11, w1, w3); DP_ACC(12, wp, w0); } }
			// "literal + rep0" (:562-597) last: it is pushed only if literal / short rep did not take slot c + 1.  It comes
			// before this worker starts node c + W (near_old and wait_deadlines rely on that).  In the reference it precedes
			// the node's other classes, so it wins ties against their entries; against older nodes' entries it loses them.
			if (lr_len != 0) {
				uint32_t nv;
				__syncwarp();
				for (;;) {
					nv = __shfl_sync(WFULL, S.nil_node, 0);
					if ((nv >> 17) == (want >> 16) && ((nv >> 1) & 0xFFFF) >= c) break;
					if (__shfl_sync(WFULL, (uint32_t)(S.seg_epoch != my_epoch || S.m_exit), 0)) { gone = true; break; }
				}
				if (gone) break;
				// the flag of node c itself; a later value means the chain warp is already past c + 1: read ours from the link
				bool nil;
				DP_ACQUIRE();
				if (((nv >> 1) & 0xFFFF) == c) nil = (nv & 1) != 0;
				else { const uint32_t m1 = S.o_meta[c + 1]; nil = DP_FLAGS(m1) == 0 && DP_D1(m1) == 1; }
				if (!nil) {
					const uint32_t c1 = S.n_c1[k];
					const uint32_t psn = (pos + 1) & H.pos_mask;
					const uint32_t pr_ = c1 + S.pb[DpEnc::st_lit(st)][psn][1].x + H.len_price(1, lr_len, psn);
					const uint32_t offset = c + 1 + lr_len;
					if (lane == 0) {
						DP_CNTA(60);
						// only for a pushed candidate: len_end decides where the segment ends
						const uint32_t le_was = atomicMax(&S.len_end_sh, offset);
						if (le_was <= c + 1) DP_CNTA(61);   // without it the segment would end at c + 1
						(void)le_was;
						uint4 *s = &rg[offset & rmask];
						const uint4 old = *s;
						if (pr_ < old.x || (pr_ == old.x && DP_SRC(offset, old.z) == c))
							*s = make_uint4(pr_, 0, DP_META(lr_len, 1u, 0u, (uint32_t)(b - hr[0] - 1)[1 + lr_len]), 0);
					}
				}
				__syncwarp(); DP_RELEASE();
				if (lane == 0) dp_sts64(&S.lr[c & 31], make_uint2(want + 1, 0u));
			}
		}
		// this segment is over for this worker: wait until the chain warp says so, then report idle
		while (S.seg_stop == DP_NONE && S.seg_epoch == my_epoch && !S.m_exit) __nanosleep(50);
		__syncwarp(); __threadfence_block();
		if (lane == 0) S.idle[w] = my_epoch;
	}
}
