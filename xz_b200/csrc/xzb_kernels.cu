// xzb_kernels.cu -- sm_90a kernels and host orchestration of the LZMA2 block path,
// exported through the C ABI in include/xzb200.h.
//
// Pipeline for a wave of B independent .xz blocks resident in HBM:
//   xzb_k_hash_keys   1 thread / position   : hash-2/3/main keys, (block,key) sort keys
//   radix sort + xzb_k_prev                 : previous occurrence per hash = the hash heads
//   xzb_k_hc | xzb_k_bt                     : match finder -> match store (HBM)
//   xzb_k_crc                               : CRC64/CRC32 of every block (slice + GF(2) fold)
//   xzb_k_parse_dp | xzb_k_parse_fast  1 CUDA block / .xz block : parser + range coder + LZMA2 chunker
//   xzb_k_finalize    1 CUDA block / .xz block : header, padding, check | raw fallback
//   xzb_k_pack_streams  1 CUDA block / .xz block : the finished Block to its place (+ Stream framing for one-shot items)
// Decode: xzb_k_decode (1 CUDA block / .xz block) + xzb_k_crc over the output; the device-resident batch adds
// xzb_k_dec_scan / xzb_k_dec_prep / xzb_k_dec_settle / xzb_k_dec_results, which read the container on the GPU.
// There is deliberately no CPU path in this file.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/xzb200.h"
#include "xzb_common.cuh"
#include "xzb_mf.cuh"
#include "xzb_dec.cuh"
#include "xzb_dec_warp.cuh"
#include "xzb_sha256.cuh"
#include "xzb_frame.cuh"
#include "xzb_dec_stream.cuh"
#include "xzb_filters.cuh"
#include "xzb_params.h"
#include "xzb_parse_warp.cuh"
#include "xzb_parse_dp.cuh"

// ------------------------------------------------------------------------------------
// Kernels
// ------------------------------------------------------------------------------------

// Wave layout (xzb_params.h): Block b's positions are [off[b], off[b] + n_b) of every per-position array, off[b] a
// multiple of 256; tile_block[t] is the Block that positions [256 t, 256 t + 256) belong to.
// One thread per position of the wave, 256-position tiles.  Keys are (block << hbits) | hash; positions that are never
// inserted (short tail, lz_encoder_mf.c:190-201, and the padding behind a Block) get the out-of-range block index B so
// that they sort behind every real key.
__global__ void __launch_bounds__(256)
xzb_k_hash_keys(const XzbMfBlock *__restrict__ blocks, const uint32_t *__restrict__ tile_block, const uint32_t *__restrict__ off, uint32_t B,
		XzbParams P, const uint32_t *__restrict__ crc, uint32_t hbm,
		uint32_t *__restrict__ keys_m, uint32_t *__restrict__ keys_2, uint32_t *__restrict__ keys_3,
		uint32_t *__restrict__ vals, uint32_t *__restrict__ mh)
{
	const uint32_t blk = tile_block[blockIdx.x];
	const size_t g = (size_t)blockIdx.x * 256 + threadIdx.x;
	const uint32_t p = (uint32_t)(g - off[blk]);
	const uint32_t n = blocks[blk].n;
	uint32_t km = B << hbm, k2 = B << 10, k3 = B << 16;
	if (p < n && n - p >= P.hash_bytes) {
		uint32_t h2 = 0, h3 = 0;
		const uint32_t hm = xzb_hash(blocks[blk].buf + p, P, crc, &h2, &h3);
		km = (blk << hbm) | hm; k2 = (blk << 10) | h2; k3 = (blk << 16) | h3;
	} else if (p < n) {
		mh[g] = 0;
	}
	keys_m[g] = km;
	if (P.hash_bytes >= 3) keys_2[g] = k2;
	if (P.hash_bytes >= 4) keys_3[g] = k3;
	vals[g] = p;
}

// After a stable sort by key: previous element with the same key is the hash head the
// reference would have read (lz_encoder_mf.c:372-379).
__global__ void __launch_bounds__(256)
xzb_k_prev(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals, size_t N, uint32_t hb, uint32_t B, const uint32_t *__restrict__ off,
		uint32_t *__restrict__ prev)
{
	const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= N) return;
	const uint32_t k = keys[i];
	const uint32_t blk = k >> hb;
	if (blk >= B) return;
	const uint32_t p = vals[i];
	uint32_t q = XZB_NONE;
	if (i > 0 && keys[i - 1] == k) q = vals[i - 1];
	prev[(size_t)off[blk] + p] = q;
}

// Binary-tree work units.  A "run" is the positions of one hash bucket (same block, same hash)
// that fall into one SEGMENT of 2^seg_shift block positions; runs of segment s only depend on runs
// of segment s-1 of the same bucket, so the match finder can publish "every block is finished up
// to position (s+1) << seg_shift" after each segment and the parser starts while later segments
// are still being searched (see encode_wave).
static const uint32_t XZB_RUN_LEN_BITS = 21;  // run length <= 2^seg_shift <= 2^20

struct XzbRunStartOp {
	const uint32_t *keys, *vals;
	uint32_t sentinel_min, seg_shift;
	__device__ bool operator()(uint32_t i) const
	{
		const uint32_t k = keys[i];
		if (k >= sentinel_min) return false;
		if (i == 0 || keys[i - 1] != k) return true;
		return (vals[i - 1] >> seg_shift) != (vals[i] >> seg_shift);
	}
};

// run_key = (segments-from-the-end << 21) | length: a DESCENDING sort puts segment 0 first and
// the longest runs of every segment at its front.
__global__ void __launch_bounds__(256)
xzb_k_run_key(const uint32_t *__restrict__ run_start, const uint32_t *__restrict__ num_runs, uint32_t n_valid,
		const uint32_t *__restrict__ vals, uint32_t seg_shift, uint32_t nseg, uint32_t *__restrict__ run_key)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t nr = *num_runs;
	if (r >= nr) return;
	const uint32_t s = run_start[r];
	const uint32_t end = r + 1 < nr ? run_start[r + 1] : n_valid;
	const uint32_t seg = vals[s] >> seg_shift;
	run_key[r] = ((nseg - 1 - seg) << XZB_RUN_LEN_BITS) | (end - s);
}

// seg_first[s] = index of the first sorted run of segment s (seg_first[nseg] = number of runs)
__global__ void __launch_bounds__(256)
xzb_k_seg_bounds(const uint32_t *__restrict__ run_key_s, const uint32_t *__restrict__ num_runs, uint32_t nseg, uint32_t *__restrict__ seg_first)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t nr = *num_runs;
	if (nr == 0) {
		if (r == 0) for (uint32_t s = 0; s <= nseg; ++s) seg_first[s] = 0;
		return;
	}
	if (r >= nr) return;
	const uint32_t seg = nseg - 1 - (run_key_s[r] >> XZB_RUN_LEN_BITS);
	const uint32_t from = r == 0 ? 0 : nseg - (run_key_s[r - 1] >> XZB_RUN_LEN_BITS);  // previous run's segment + 1
	for (uint32_t s = from; s <= seg; ++s) seg_first[s] = r;
	if (r == nr - 1) for (uint32_t s = seg + 1; s <= nseg; ++s) seg_first[s] = nr;
}

// "all blocks are searched up to (exclusive) block position `value`" -- read by the parser (mf_wait)
__global__ void xzb_k_publish(uint32_t *flag, uint32_t value)
{
	__threadfence();
	*(volatile uint32_t *)flag = value;
}

// Hash chain: one thread per position of the wave, 128-position tiles (half a tile of tile_block).
__global__ void __launch_bounds__(128)
xzb_k_hc(const XzbMfBlock *__restrict__ blocks, const uint32_t *__restrict__ tile_block, const uint32_t *__restrict__ off, XzbParams P)
{
	const size_t g = (size_t)blockIdx.x * 128 + threadIdx.x;
	const uint32_t blk = tile_block[blockIdx.x >> 1];
	const XzbMfBlock B = blocks[blk];
	const uint32_t p = (uint32_t)(g - off[blk]);
	if (p >= B.n) return;
	xzb_hc_position(B, P, p);
}

// Binary tree, one segment: persistent threads pull runs (longest first) from the segment's work
// counter and replay the bucket's tree insertions in position order.
__global__ void __launch_bounds__(128)
xzb_k_bt(const XzbMfBlock *__restrict__ blocks, XzbParams P, const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
		const uint32_t *__restrict__ run_start, const uint32_t *__restrict__ run_key, const uint32_t *__restrict__ seg_first,
		uint32_t seg, uint32_t hb, uint32_t *counters, const uint32_t *parser_sm, uint32_t live_ctas)
{
	// While the parser kernel is resident, its SMs are left alone: a CTA that lands on one of them
	// retires at once (the launch is oversubscribed by that many CTAs), so the parser's critical
	// warp does not share issue slots or L1 with the search.  parser_sm == nullptr: use every SM.
	if (parser_sm != nullptr) {
		uint32_t smid;
		asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
		if (smid < 256 && ((const volatile uint32_t *)parser_sm)[smid] != 0) return;
	}
	const uint32_t lo = seg_first[seg];
	const uint32_t nr = seg_first[seg + 1] - lo;
	// Runs are sorted longest first and handed out by one work counter.  The first T tickets are
	// permuted lane-major (a warp's 32 simultaneous tickets c..c+31 become runs lane * NW + c / 32), so
	// the heaviest buckets land on DIFFERENT warps: 32 long serial chains inside one warp would
	// time-share a single instruction stream.  The permutation is a bijection on [0, T) whatever
	// number of CTAs actually takes part.
	const uint32_t T = live_ctas * blockDim.x, NW = T >> 5;
	for (;;) {
		const uint32_t c = atomicAdd(counters + seg, 1u);
		const uint32_t r = c < T ? (c & 31) * NW + (c >> 5) : c;
		if (c >= T && r >= nr) return;
		if (r >= nr) continue;
		const uint32_t s = run_start[lo + r];
		const uint32_t L = run_key[lo + r] & ((1u << XZB_RUN_LEN_BITS) - 1);
		const uint32_t k = keys[s];
		const XzbMfBlock B = blocks[k >> hb];
		// the bucket's last position in an earlier segment is the hash head of this run's first position
		uint32_t prev = (s > 0 && keys[s - 1] == k) ? vals[s - 1] : XZB_NONE;
		for (uint32_t i = 0; i < L; ++i) {
			const uint32_t p = vals[s + i];
			xzb_bt_position(B, P, p, prev);
			prev = p;
		}
	}
}

// CRC of each block: slice 0 (short) starts from the real init value, the other slices from
// zero; Z = "advance the register over L zero bytes" as a 64x64 GF(2) matrix (one column per
// thread), then thread 0 folds the slices left to right.  Reflected CRC, check/crc64_fast.c
// and crc32_fast.c compute the same polynomial division.  count (when given): the number of jobs, in device memory, for
// a launch sized before it was known; CTAs past it return.
struct XzbCrcJob { const uint8_t *data; uint32_t size; };

__global__ void __launch_bounds__(1024)
xzb_k_crc(const XzbCrcJob *__restrict__ jobs, const uint64_t *__restrict__ table, uint64_t init, uint64_t *__restrict__ out, uint32_t out_stride,
		const uint32_t *count)
{
	__shared__ uint64_t s_tab[256];
	__shared__ uint64_t s_part[1024];
	__shared__ uint64_t s_z[64];
	if (count != nullptr && blockIdx.x >= *count) return;
	const XzbCrcJob job = jobs[blockIdx.x];
	const uint32_t T = blockDim.x;
	const uint32_t t = threadIdx.x;
	for (uint32_t i = t; i < 256; i += T) s_tab[i] = table[i];
	__syncthreads();
	const uint32_t n = job.size;
	const uint32_t L = n == 0 ? 1 : (n + (T - 2)) / (T - 1);  // ceil(n / (T-1))
	const uint32_t k = n / L;                                  // full slices, k <= T-1
	const uint32_t r = n - k * L;                              // leading short slice
	uint64_t c = 0;
	if (t <= k) {
		uint32_t beg, len;
		if (t == 0) { beg = 0; len = r; c = init; } else { beg = r + (t - 1) * L; len = L; }
		const uint8_t *d = job.data + beg;
		for (uint32_t i = 0; i < len; ++i) c = s_tab[(c ^ d[i]) & 0xFF] ^ (c >> 8);
	}
	s_part[t] = c;
	if (t >= T - 64) {  // the last 64 threads are idle whenever k < T-64; otherwise they do both jobs
		const uint32_t j = t - (T - 64);
		uint64_t z = 1ull << j;
		for (uint32_t i = 0; i < L; ++i) z = s_tab[z & 0xFF] ^ (z >> 8);
		s_z[j] = z;
	}
	__syncthreads();
	if (t == 0) {
		uint64_t st = s_part[0];
		for (uint32_t i = 1; i <= k; ++i) {
			uint64_t adv = 0;
			for (uint32_t j = 0; j < 64; ++j) if ((st >> j) & 1) adv ^= s_z[j];
			st = adv ^ s_part[i];
		}
		out[(size_t)blockIdx.x * out_stride] = st ^ init;  // final xor == init for both CRC-32 and CRC-64/XZ
	}
}

// SHA-256 of each block (LZMA_CHECK_SHA256): thread 0 of CTA b hashes block b; the chain is serial per
// message, the wave's blocks give the parallelism.  out: 32 bytes per block.  count: as for xzb_k_crc.
__global__ void __launch_bounds__(32)
xzb_k_sha256(const XzbCrcJob *__restrict__ jobs, uint8_t *__restrict__ out, const uint32_t *count)
{
	if (threadIdx.x != 0 || (count != nullptr && blockIdx.x >= *count)) return;
	const XzbCrcJob job = jobs[blockIdx.x];
	uint8_t digest[32];
	xzb_sha256(job.data, job.size, digest);
	for (int i = 0; i < 32; ++i) out[(size_t)blockIdx.x * 32 + i] = digest[i];
}

struct XzbEncJob {
	const uint8_t *in;
	uint32_t in_size;
	uint8_t *out;            // per-block scratch
	uint32_t out_cap;
	uint32_t header_size;    // reserved from the maximum sizes (stream_encoder_mt.c:225-237)
	uint32_t oneshot;        // 1 = lzma_block_buffer_encode() framing (block_buffer_encoder.c:165-281)
	uint64_t fit_limit;      // see xzb_block_finish_normal
};

// Parser kernels: one CUDA block per .xz block, all coder state in shared memory (xzb_parse_warp.cuh,
// xzb_parse_dp.cuh).  The coding warp and the warps that work for it share these parameters.
template <class ENC>
static __device__ void xzb_setup_warp(ENC &E, const XzbEncJob &job, const XzbMfBlock &blk, const XzbParams &P)
{
	E.buf = blk.buf; E.size = job.in_size;   // the bytes LZMA2 codes (after Delta / BCJ); job.in stays the unfiltered input
	E.g_mh = blk.mh; E.g_mp = blk.mp; E.g_ovf = blk.ovf;
	E.read_pos = 0; E.read_ahead = 0; E.ring_base = 0x80000000u;
	E.nice_len = P.nice_len;
	E.pos_mask = (1u << P.pb) - 1; E.lc = P.lc; E.literal_mask = (0x100u << P.lp) - (0x100u >> P.lc);
	E.dist_table_size = P.dist_table_size; E.len_table_size = P.len_table_size; E.num_pos_states = 1u << P.pb;
	E.uncomp_size = 0; E.is_initialized = 0; E.n_symbols = 0; E.matches_count = 0; E.longest_match_length = 0;
	E.rc_out = job.out; E.rc_out_pos = 0;
}

// Dynamic shared memory of the two-warp fast-mode form.  Its state needs only sizeof(FS<false>), but each Block of a wave
// that leaves SMs idle gets an SM to itself: more than half of an SM's 228 KB leaves no room for a second parser CTA, so
// the B parser CTAs take B SMs and the match finder beside them counts on the other sm_count - B (`avoid`, encode_wave).
// Above 196 KB the SM also keeps the shared-memory / L1 split that the normal-mode kernel (sizeof(DS)) runs with.
#define XZB_SOLO_SMEM (220u * 1024u)

// Fast mode (presets 0-3): three warps per .xz Block.
//   warp 1  decisions: lzma_lzma_optimum_fast looks only at the match store, the window and the reps, so it runs ahead;
//   warp 0  coding: resolves every symbol's probability indices in closed form, adapts the probabilities, LZMA2 chunker;
//   warp 2  CODER_WARP: range coder arithmetic + byte output (xzb_w_coder_main), fed through a ring of (probability, bit)
//           records; otherwise warp 0 runs the range coder itself and warp 2 returns at once.
// The host picks the form per wave (see launch_parse).  The coder-warp form is launched with sizeof(FS<true>), so several
// Blocks share an SM; the two-warp form with XZB_SOLO_SMEM.
template <bool CODER_WARP>
__global__ void __launch_bounds__(96)
xzb_k_parse_fast(const XzbEncJob *__restrict__ jobs, const XzbMfBlock *__restrict__ blocks, XzbParams P,
		const uint32_t *mf_flag, uint32_t *parser_sm, uint64_t mf_stall_ns, XzbBlockResult *__restrict__ results, uint32_t *__restrict__ payload_end)
{
	extern __shared__ __align__(16) uint8_t xzb_smem[];
	FS<CODER_WARP> &S = *reinterpret_cast<FS<CODER_WARP> *>(xzb_smem);
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t warp = threadIdx.x >> 5;
	const uint32_t b = blockIdx.x;
	const XzbEncJob job = jobs[b];
	if (threadIdx.x == 0) {
		uint32_t smid;
		asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
		if (smid < 256) ((volatile uint32_t *)parser_sm)[smid] = 1;  // the match finder's CTAs keep off this SM (xzb_k_bt)
	}
	if (threadIdx.x < XZB_FRING) S.f_tag[threadIdx.x] = 0;
	if (threadIdx.x == 0) {
		S.f_epoch = 0; S.f_start_pos = 0; S.f_consumed = 0; S.m_exit = 0;
		S.rcq_head = 0; S.rcq_tail = 0; S.rcq_T = 1; S.rcq_flushes = 0; S.rcq_out_pos = 0; S.rcq_out = nullptr;
	}
	__syncthreads();
	WarpEncT<FS<CODER_WARP>> E(S, lane);
	xzb_setup_warp(E, job, blocks[b], P);
	E.mf_flag = mf_flag; E.mf_done = 0; E.mf_stall_ns = mf_stall_ns;
	if (warp == 1) { xzb_w_fast_parser_main(S, E); return; }
	if (warp == 2) {
		if constexpr (CODER_WARP) xzb_w_coder_main(S, E);
		return;
	}
	E.reset();
	uint32_t out_pos = job.header_size, ncl = 0, ncr = 0;
	const int ret = xzb_w_lzma2_encode_block(E, P, job.out, job.out_cap, &out_pos, &ncl, &ncr);
	if (lane == 0) {
		S.m_exit = 1;
		XzbBlockResult *res = results + b;
		res->ret = (uint32_t)ret;
		res->n_symbols = E.n_symbols; res->n_chunks_lzma = ncl; res->n_chunks_raw = ncr;
		payload_end[b] = out_pos;
	}
}

// Normal mode (presets 4-9): dataflow-DP parser of xzb_parse_dp.cuh.  Warp 0 = chain warp (DP recurrence, probability
// adaptation, LZMA2 chunker), warp 1 = gather warp, warp 2 = coder warp (range coder arithmetic + byte output),
// the other warps off sub-partition 0 = workers (W = 10, or 3 when nice_len > 127).
// trace (debugging aid, XZB_TRACE): block 0 records (position, back, len) of every symbol; trace[-1] = count.
// The chain warp has a scheduler of its own: warps 4, 8, 12 (same SM sub-partition as warp 0) retire at once, so the
// critical warp shares neither issue slots nor the sub-partition's instruction cache with the team's much larger code.
__global__ void __launch_bounds__(512, 1)
xzb_k_parse_dp(const XzbEncJob *__restrict__ jobs, const XzbMfBlock *__restrict__ blocks, XzbParams P,
		const uint8_t *__restrict__ price_table, const uint32_t *mf_flag, uint32_t *parser_sm, uint64_t mf_stall_ns,
		XzbBlockResult *__restrict__ results, uint32_t *__restrict__ payload_end, uint32_t *trace, uint32_t trace_cap)
{
	extern __shared__ __align__(16) uint8_t xzb_smem[];
	DS &S = *reinterpret_cast<DS *>(xzb_smem);
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t warp = threadIdx.x >> 5;
	const uint32_t b = blockIdx.x;
	const XzbEncJob job = jobs[b];
	for (uint32_t i = threadIdx.x; i < 128; i += blockDim.x) S.prices[i] = price_table[i];
	if (threadIdx.x == 0) {
		uint32_t smid;
		asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
		if (smid < 256) ((volatile uint32_t *)parser_sm)[smid] = 1;  // the match finder's CTAs keep off this SM (xzb_k_bt)
		S.seg_epoch = 0; S.seg_P0 = 0; S.seg_position0 = 0; S.fin_node = 0; S.nil_node = 0; S.seg_stop = DP_NONE; S.m_exit = 0; S.len_end_sh = 0;
		S.rcq_head = 0; S.rcq_tail = 0; S.rcq_T = 1; S.rcq_flushes = 0; S.rcq_out_pos = 0; S.rcq_out = nullptr;
	}
	if (threadIdx.x < 32) S.prep[threadIdx.x] = make_uint4(0u, 0u, 0u, 0u);
	if (threadIdx.x <= DP_WMAX) S.idle[threadIdx.x] = 0;
	if (threadIdx.x < 32) { S.part_tag[threadIdx.x] = 0; S.res_c[threadIdx.x] = make_uint4(0u, 0u, 0u, 0u); }
#ifdef XZB_DP_PROF
	if (threadIdx.x < 32) S.prof[threadIdx.x] = 0;
#endif
	for (uint32_t i = threadIdx.x; i < DP_NR; i += blockDim.x) S.ph[i] = 0;
	__syncthreads();
	DpEnc E(S, lane);
	xzb_setup_warp(E, job, blocks[b], P);
	E.mf_flag = mf_flag; E.mf_done = 0; E.mf_stall_ns = mf_stall_ns;
	if (warp != 0 && (warp & 3) == 0) return;   // see above
	const uint32_t nwarps = blockDim.x / 32;
	E.W = nwarps - 3 - (nwarps - 1) / 4;
	E.rsize = P.nice_len > 127 ? 1024u : 256u;
	E.rmask = E.rsize - 1; E.rstride = E.rsize + 1;
	E.plain_stride = P.nice_len > 127 ? 272u : 128u;
	E.epoch = 0;
	E.sym_cur = E.sym_end = 0;
	E.trace = (b == 0) ? trace : nullptr; E.trace_cap = trace_cap; E.trace_n = 0;
	if (warp == 1) { xzb_dp_gather_main(S, E); return; }
	if (warp == 2) { xzb_dp_coder_main(S, E); return; }
	if (warp != 0) { xzb_dp_worker_main(S, E, warp - 3 - (warp >> 2)); return; }
#ifdef XZB_DP_PROF
	const long long k_t0 = clock64();
	unsigned long long k_ns0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(k_ns0));
#endif
	E.reset();
	uint32_t out_pos = job.header_size, ncl = 0, ncr = 0;
	const int ret = xzb_w_lzma2_encode_block(E, P, job.out, job.out_cap, &out_pos, &ncl, &ncr);
	if (lane == 0) {
		S.m_exit = 1;
		XzbBlockResult *res = results + b;
		res->ret = (uint32_t)ret;
		res->n_symbols = E.n_symbols; res->n_chunks_lzma = ncl; res->n_chunks_raw = ncr;
		payload_end[b] = out_pos;
		if (E.trace != nullptr) E.trace[-1] = E.trace_n < trace_cap ? E.trace_n : trace_cap;
#ifdef XZB_DP_PROF
		if (b == 0) {
			unsigned long long k_ns1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(k_ns1));
			const double cyc = (double)(clock64() - k_t0), k_ns = (double)(k_ns1 - k_ns0);
			printf("DPPROF chain warp: %.0f Mcycles in %.1f ms = %.0f MHz; %.0f cycles per node, all included; look-ahead hits %.1f%% (literal/short rep won %.1f%%, record late %.1f%%, other candidate %.1f%%)\n", cyc / 1e6, k_ns / 1e6, cyc / k_ns * 1e3, cyc / ((double)S.prof[4] + 1e-9), 100.0 * (double)S.prof[20] / ((double)S.prof[4] + 1e-9),
				100.0 * (double)S.prof[23] / ((double)S.prof[4] + 1e-9), 100.0 * (double)S.prof[22] / ((double)S.prof[4] + 1e-9), 100.0 * (double)S.prof[21] / ((double)S.prof[4] + 1e-9));
			const double n = (double)S.prof[4] + 1e-9, nw = (double)S.prof[10] + 1e-9;
			printf("DPPROF nodes %llu: prep_wait %.0f derive+lit+publish %.0f deadline_wait %.0f gather+combine %.0f cyc/node; slow-path %llu x %.0f cyc | worker0 nodes %llu: fin_wait %.0f fin->ph1 %.0f fin->ph3 %.0f prep %.0f\n",
				S.prof[4], S.prof[0] / n, S.prof[1] / n, S.prof[2] / n, S.prof[3] / n, S.prof[6], S.prof[5] / ((double)S.prof[6] + 1e-9),
				S.prof[10], S.prof[8] / nw, S.prof[9] / nw, S.prof[11] / nw, S.prof[12] / nw);
			printf("DPPROF loop top + instrumentation: %.0f cyc/node; worker0 near path (node final seen -> near candidates pushed): %.0f cyc x %llu\n",
				(double)S.prof[7] / ((double)S.prof[4] + 1e-9), (double)S.prof[29] / ((double)S.prof[30] + 1e-9), S.prof[30]);
			printf("DPPROF gather: slots that had to wait for node t-2: %llu, t-3: %llu, t-4: %llu, t-5..8: %llu, older: %llu\n", S.prof[24], S.prof[25], S.prof[26], S.prof[27], S.prof[28]);
			const double ns = (double)S.prof[15] + 1e-9, ng = (double)S.prof[19] + 1e-9;
			printf("DPPROF symbols %llu: optimum_normal %.0f encode_symbol %.0f cyc/symbol | segments %llu: helper1 %.0f idle_wait %.0f backward %.0f cyc/segment\n",
				S.prof[15], S.prof[13] / ns, S.prof[14] / ns, S.prof[19], S.prof[16] / ng, S.prof[17] / ng, S.prof[18] / ng);
		}
#endif
	}
}

__global__ void __launch_bounds__(256)
xzb_k_finalize(const XzbEncJob *__restrict__ jobs, const uint32_t *__restrict__ crc32_table, XzbParams P, uint32_t check,
		const uint8_t *__restrict__ check_bytes /* 32 per block: little-endian CRC or SHA-256 */, const uint32_t *__restrict__ payload_end,
		XzbBlockResult *__restrict__ results)
{
	__shared__ int s_fallback;
	const uint32_t b = blockIdx.x;
	const XzbEncJob job = jobs[b];
	XzbBlockResult *res = results + b;
	if (res->ret == XZB_MF_STALL) return;  // the host parses this wave again (encode_wave)
	if (threadIdx.x == 0) {
		bool ok = false;
		if (res->ret == XZB_OK)
			ok = xzb_block_finish_normal(crc32_table, job.out, payload_end[b], job.header_size, job.fit_limit, job.oneshot, check,
					check_bytes + (size_t)b * 32, job.in_size, P.dict_prop, res, P.ff, P.ff_len, P.n_pre);
		// XZB_BUF_ERROR from the chunker only means "take the fallback"; anything else is an encoder failure and stays
		const bool internal = res->ret != XZB_OK && res->ret != XZB_BUF_ERROR;
		if (!internal) res->ret = XZB_OK;
		s_fallback = !ok && !internal;
	}
	__syncthreads();
	if (s_fallback)
		xzb_block_finish_raw(crc32_table, job.in, job.in_size, job.out, check, check_bytes + (size_t)b * 32, res, threadIdx.x, blockDim.x);
}

// Places finished Blocks: one CTA per job copies its Block out of scratch to `dst`; with `frame` the job becomes a whole
// one-shot Stream (xzb_pack_stream).  src == nullptr with frame: the Stream with no Block.
struct XzbPackJob {
	const uint8_t *src;
	uint8_t *dst;
	uint64_t unpadded, uncomp;
	uint32_t size, frame;
};

__global__ void __launch_bounds__(256)
xzb_k_pack_streams(const XzbPackJob *__restrict__ jobs, const uint32_t *__restrict__ crc32_table, uint32_t check)
{
	const XzbPackJob j = jobs[blockIdx.x];
	xzb_pack_stream(crc32_table, j.dst, j.src, j.size, j.unpadded, j.uncomp, check, j.frame != 0, threadIdx.x, blockDim.x);
}

// ---- Delta / BCJ filters over whole Blocks (xzb_filters.cuh) ----
// One CUDA block per .xz Block and chain stage.  `src != dst` only for the Delta encoder (out of place, so every
// byte reads its unfiltered predecessor); everything else works in place on `dst`.
struct XzbFiltJob {
	const uint8_t *src;
	uint8_t *dst;
	uint32_t size, id, arg, pad_;
};

__global__ void __launch_bounds__(256)
xzb_k_filter(const XzbFiltJob *__restrict__ jobs, int enc)
{
	__shared__ uint32_t s_sum[256];
	const XzbFiltJob j = jobs[blockIdx.x];
	const uint32_t tid = threadIdx.x, nt = blockDim.x;
	if (j.size == 0) return;
	if (j.id == XZB_FILTER_DELTA) {
		const uint32_t d = j.arg;
		if (enc) {   // delta_encoder.c:20-46
			for (uint32_t i = tid; i < j.size; i += nt) j.dst[i] = (uint8_t)(j.src[i] - (i >= d ? j.src[i - d] : 0u));
			return;
		}
		// delta_decoder.c:20-33: out[i] = in[i] + out[i - d] is a running sum (mod 256) along each residue class of i mod d;
		// thread t takes segment t / d of class t % d: local sums, exclusive scan over the segments of the class, second pass
		const uint32_t cls = tid % d, nseg = nt / d, seg = tid / d;   // threads with seg >= nseg idle (nt not a multiple of d)
		const uint32_t n_cls = cls < j.size ? (j.size - cls + d - 1) / d : 0;   // elements of this class
		const uint32_t per = nseg ? (n_cls + nseg - 1) / nseg : 0;
		const uint32_t e0 = seg < nseg ? (uint32_t)min((uint64_t)seg * per, (uint64_t)n_cls) : 0;
		const uint32_t e1 = seg < nseg ? (uint32_t)min((uint64_t)(seg + 1) * per, (uint64_t)n_cls) : 0;
		uint32_t sum = 0;
		for (uint32_t e = e0; e < e1; ++e) sum += j.dst[cls + e * d];
		s_sum[tid] = sum & 0xFF;
		__syncthreads();
		uint32_t run = 0;
		for (uint32_t k = 0; k < seg && k < nseg; ++k) run += s_sum[k * d + cls];
		for (uint32_t e = e0; e < e1; ++e) { run += j.dst[cls + e * d]; j.dst[cls + e * d] = (uint8_t)run; }
		return;
	}
	const uint32_t unit = xzb_filter_unit(j.id);
	if (unit != 0) {   // independent units: one per thread
		const uint32_t n = j.size / unit;
		for (uint32_t u = tid; u < n; u += nt) xzb_bcj_unit(j.id, j.dst + (size_t)u * unit, j.arg + u * unit, enc != 0);
		return;
	}
	if (tid == 0) {    // x86 / ARM-Thumb: the position of the next unit depends on the previous conversion
		if (j.id == XZB_FILTER_X86) xzb_bcj_x86(j.dst, j.size, j.arg, enc != 0);
		else if (j.id == XZB_FILTER_ARMTHUMB) xzb_bcj_armthumb(j.dst, j.size, j.arg, enc != 0);
		else if (j.id == XZB_FILTER_RISCV) xzb_bcj_riscv(j.dst, j.size, j.arg, enc != 0);
	}
}

struct XzbDecJob {
	const uint8_t *in;
	uint32_t in_size;
	uint8_t *out;
	uint32_t out_limit;
	uint32_t dict_size;
};

// One warp per .xz block; the probability model lives in shared memory (28 KB, so several blocks
// share an SM), every lane runs the (inherently serial) bit decoding uniformly, lane 0 stores
// literals and all lanes share match / raw-chunk copies.
__global__ void __launch_bounds__(32)
xzb_k_decode(const XzbDecJob *__restrict__ jobs, XzbDecResult *__restrict__ results)
{
	extern __shared__ __align__(16) uint8_t xzb_smem[];
	XzbDec *d = reinterpret_cast<XzbDec *>(xzb_smem);
	const uint32_t b = blockIdx.x;
	const XzbDecJob job = jobs[b];
	uint32_t iu = 0, ou = 0;
	const int ret = xzb_lzma2_decode(d, job.in, job.in_size, job.dict_size, job.out, job.out_limit, &iu, &ou, threadIdx.x, 32);
	if (threadIdx.x == 0) { results[b].ret = (uint32_t)ret; results[b].in_used = iu; results[b].out_used = ou; }
}

// ---- device-resident Stream decode (xzb_stream_buffer_decode_batch_device) ----
// Each round: xzb_k_dec_scan (the next run of every unfinished item, xzb_dec_scan) -> xzb_k_decode over the run's
// Blocks -> xzb_k_dec_prep (filter and check job lists) -> xzb_k_filter per chain level -> xzb_k_crc / xzb_k_sha256
// -> xzb_k_dec_settle (xzb_dec_settle, and xzb_dec_end at the Index).  The cursors stay in HBM between rounds.
struct XzbDecItem {             // item i of a group: its Stream, its output slot, its Index record area
	const uint8_t *in;
	uint8_t *out;
	xzb_index_record *recs;
	uint64_t rec_cap;
};
struct XzbDecRound { uint32_t job0, nb, chk0, pad_; };   // the item's run in the round's job list; its first check job
struct XzbDecCounters {
	uint32_t njobs;             // jobs asked for (may exceed the round's capacity; the grants stop there)
	uint32_t depth;             // longest Delta / BCJ chain in front of LZMA2 among the round's Blocks
	uint32_t checks;            // check lists in use: 1 CRC32, 2 CRC64, 4 SHA-256
	uint32_t live;              // items not finished after xzb_k_dec_settle
	uint32_t nchk[3];           // jobs of the CRC32, CRC64 and SHA-256 lists
	uint32_t pad_;
	unsigned long long positions;  // bytes of the validated Blocks (kept over the rounds)
};
struct XzbDecOut { uint64_t out_size, in_used; uint32_t ret, pad_; };

XZB_HD uint32_t xzb_dec_check_list(uint32_t check) { return check == 1 ? 0 : check == 4 ? 1 : 2; }

// One thread per item.  The run is scanned twice: once to learn its length, which reserves that many job slots, and
// again into the slots granted (a prefix of the run when the round's capacity runs out; the rest waits a round).
__global__ void __launch_bounds__(128)
xzb_k_dec_scan(XzbDecCursor *__restrict__ cur, const XzbDecItem *__restrict__ items, uint32_t n, const uint32_t *__restrict__ crc32_table,
		uint32_t cap, XzbDecBlk *__restrict__ blks, XzbDecJob *__restrict__ jobs, XzbDecRound *__restrict__ round, XzbDecCounters *cnt)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	round[i].nb = 0;
	if (cur[i].done) return;
	const XzbDecItem it = items[i];
	XzbDecCursor c = cur[i];
	const uint32_t want = xzb_dec_scan(c, it.in, crc32_table, nullptr, cap, it.recs);
	if (want == 0) { cur[i] = c; return; }   // finished by its header or at its Index
	const uint32_t base = atomicAdd(&cnt->njobs, want);
	if (base >= cap) return;
	c = cur[i];
	const uint32_t nb = xzb_dec_scan(c, it.in, crc32_table, blks + base, min(want, cap - base), it.recs);
	uint32_t depth = 0;
	for (uint32_t b = 0; b < nb; ++b) {
		const XzbDecBlk &k = blks[base + b];
		XzbDecJob j;
		j.in = it.in + k.hdr_off + k.hb.hsize; j.in_size = k.in_avail;
		j.out = it.out + k.out_off; j.out_limit = k.out_limit; j.dict_size = k.hb.dict_size;
		jobs[base + b] = j;
		depth = max(depth, k.hb.n_pre);
	}
	round[i] = XzbDecRound{ base, nb, 0, 0 };
	if (depth) atomicMax(&cnt->depth, depth);
	const uint32_t ck = xzb_dec_check_computed(c);
	if (ck) atomicOr(&cnt->checks, 1u << xzb_dec_check_list(ck));
	cur[i] = c;
}

// One thread per item of the round: the filter jobs of every chain level (in reverse chain order, size 0 where the
// Block's chain is shorter) and the item's Blocks as one stretch of its check list.
__global__ void __launch_bounds__(128)
xzb_k_dec_prep(const XzbDecCursor *__restrict__ cur, XzbDecRound *__restrict__ round, uint32_t n, const XzbDecBlk *__restrict__ blks,
		const XzbDecJob *__restrict__ jobs, const XzbDecResult *__restrict__ results, uint32_t cap, XzbFiltJob *__restrict__ filt,
		XzbCrcJob *__restrict__ chk_jobs, XzbDecCounters *cnt)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const XzbDecRound r = round[i];
	if (r.nb == 0) return;
	const uint32_t depth = cnt->depth;
	for (uint32_t b = 0; b < r.nb; ++b) {
		const uint32_t j = r.job0 + b;
		const XzbBlockHeader &hb = blks[j].hb;
		for (uint32_t lvl = 0; lvl < depth; ++lvl) {
			XzbFiltJob f{ jobs[j].out, jobs[j].out, 0, 0, 0, 0 };
			if (lvl < hb.n_pre) { const XzbPreFilter p = hb.pre[hb.n_pre - 1 - lvl]; f.size = results[j].out_used; f.id = p.id; f.arg = p.arg; }
			filt[(size_t)lvl * cap + j] = f;
		}
	}
	const uint32_t ck = xzb_dec_check_computed(cur[i]);
	if (ck == 0) return;
	const uint32_t list = xzb_dec_check_list(ck);
	const uint32_t k0 = atomicAdd(&cnt->nchk[list], r.nb);
	round[i].chk0 = k0;
	for (uint32_t b = 0; b < r.nb; ++b) chk_jobs[(size_t)list * cap + k0 + b] = XzbCrcJob{ jobs[r.job0 + b].out, results[r.job0 + b].out_used };
}

// One thread per item: xzb_dec_settle over the item's run against the checks computed for it, counting the items
// that still have Blocks to go.
__global__ void __launch_bounds__(128)
xzb_k_dec_settle(XzbDecCursor *__restrict__ cur, const XzbDecItem *__restrict__ items, const XzbDecRound *__restrict__ round, uint32_t n,
		const uint32_t *__restrict__ crc32_table, const XzbDecBlk *__restrict__ blks, const XzbDecResult *__restrict__ results, uint32_t cap,
		const uint64_t *__restrict__ crcv, const uint8_t *__restrict__ shav, XzbDecCounters *cnt)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const XzbDecRound r = round[i];
	if (r.nb == 0) { if (!cur[i].done) atomicAdd(&cnt->live, 1u); return; }
	XzbDecCursor c = cur[i];
	const XzbDecItem it = items[i];
	const uint32_t list = xzb_dec_check_list(c.check);
	const uint8_t *chk = list == 2 ? shav + 32 * (size_t)r.chk0 : (const uint8_t *)(crcv + (size_t)list * cap + r.chk0);
	const uint64_t produced = xzb_dec_settle(c, it.in, crc32_table, blks + r.job0, results + r.job0, chk, list == 2 ? 32 : 8, it.recs, it.rec_cap);
	if (produced) atomicAdd(&cnt->positions, (unsigned long long)produced);
	if (!c.done) atomicAdd(&cnt->live, 1u);
	cur[i] = c;
}

// The results with xzb_stream_buffer_decode()'s mapping: input that ended early is XZB_DATA_ERROR.
__global__ void __launch_bounds__(128)
xzb_k_dec_results(const XzbDecCursor *__restrict__ cur, uint32_t n, XzbDecOut *__restrict__ out)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const XzbDecCursor c = cur[i];
	const int code = c.ret == XZB_BUF_ERROR && c.buf_reason == 1 ? XZB_DATA_ERROR : c.ret;
	out[i] = XzbDecOut{ c.out_size, c.in_used, (uint32_t)code, 0 };
}

// ------------------------------------------------------------------------------------
// Context
// ------------------------------------------------------------------------------------
struct DevBuf {
	void *p = nullptr;
	size_t cap = 0;
};

struct xzb_ctx {
	int dec_buf_reason = 0;
	int device = 0;
	cudaStream_t stream = nullptr;
	XzbHostTables h_tab;
	uint32_t *d_crc32 = nullptr;
	uint64_t *d_crc64 = nullptr, *d_crc32w = nullptr;
	uint8_t *d_prices = nullptr;
	char err[256] = { 0 };
	xzb_stats stats;
	cudaEvent_t ev[12];
	// workspace
	DevBuf keys_a, keys_b, vals_a, vals_b, keys_2, keys_3, prev2, prev3, prevm, son, mh, mp, ovf, cub_tmp;
	DevBuf run_start, run_len, run_start_s, run_len_s, small, encs, scratch, in_stage, decs, dec_in, dec_out;
	DevBuf filt_a, filt_b, filt_jobs;   // Delta / BCJ: filtered copies of a wave's input, per-Block stage jobs
	DevBuf out_stage, pack_jobs;        // finished Blocks / Streams on their way to host memory, xzb_k_pack_streams jobs
	std::vector<XzbPreFilter> pre;      // the encoder's filters in front of LZMA2 (xzb_ctx_set_filters)
	int sm_count = 132;
	cudaStream_t stream_mf = nullptr;   // match-finder segments run here while the parser consumes them
	cudaEvent_t ev_mf[4];
	DevBuf seg_meta;                    // [0] progress flag, [1..nseg+1] seg_first, then nseg work counters
	bool overlap = true;                // XZB_OVERLAP=0, or a profiler/sanitizer that serialises kernels, turns it off
	uint32_t seg_shift = 20;            // XZB_SEG_SHIFT
	bool avoid_parser_sms = true;       // XZB_MF_AVOID_PARSER_SMS
	uint64_t mf_stall_ns = XZB_MF_STALL_NS;  // XZB_MF_STALL_MS
	uint32_t mf_stalls = 0;
	const char *trace_path = nullptr;  // XZB_TRACE=file: symbol trace of block 0 of every wave (normal mode, debugging aid)
	DevBuf trace;
	uint32_t max_wave_blocks = 0;
};

static int set_err(xzb_ctx *ctx, int code, const char *fmt, ...)
{
	va_list ap; va_start(ap, fmt);
	vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
	va_end(ap);
	return code;
}

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
	return set_err(ctx, e_ == cudaErrorMemoryAllocation ? XZB_MEM_ERROR : XZB_PROG_ERROR, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)

static int ensure(xzb_ctx *ctx, DevBuf &b, size_t size)
{
	if (b.cap >= size) return XZB_OK;
	if (b.p) { cudaFree(b.p); b.p = nullptr; b.cap = 0; }
	CK(cudaMalloc(&b.p, size));
	b.cap = size;
	return XZB_OK;
}
#define EN(buf, size) do { int r_ = ensure(ctx, buf, size); if (r_ != XZB_OK) return r_; } while (0)

static void free_buf(DevBuf &b) { if (b.p) cudaFree(b.p); b.p = nullptr; b.cap = 0; }

extern "C" int xzb_lzma_preset(xzb_lzma_options *opt, uint32_t preset) { return xzb_preset((XzbLzmaOptions *)opt, preset); }
extern "C" uint64_t xzb_block_bound(uint64_t u)
{
	// overflow rules of lzma2_bound(), block_buffer_encoder.c:31-53 (COMPRESSED_SIZE_MAX :18-21)
	const uint64_t comp_max = (((~0ull) >> 1) - 1024 - 64) & ~3ull;
	if (u > comp_max) return 0;
	const uint64_t overhead = ((u + XZB_LZMA2_CHUNK_MAX - 1) / XZB_LZMA2_CHUNK_MAX) * 3 + 1;
	if (comp_max - overhead < u) return 0;
	return xzbi_block_bound(u);
}

extern "C" uint64_t xzb_stream_bound(uint64_t in_size, uint64_t block_size)
{
	if (block_size == 0) return 0;
	const uint64_t nb = (in_size + block_size - 1) / block_size;
	return 12 + nb * xzbi_block_bound(block_size) + (8 + nb * 18 + 8) + 12;
}

extern "C" int xzb_device_count(void)
{
	int count = 0;
	return cudaGetDeviceCount(&count) == cudaSuccess ? count : 0;
}

extern "C" int xzb_ctx_create(xzb_ctx **out, int device)
{
	*out = nullptr;
	int count = 0;
	if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) {
		fprintf(stderr, "xzb200: no usable CUDA device (requested %d of %d); this library has no CPU path\n", device, count);
		return XZB_PROG_ERROR;
	}
	xzb_ctx *ctx = new xzb_ctx();
	ctx->device = device;
	memset(&ctx->stats, 0, sizeof(ctx->stats));
	if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return XZB_PROG_ERROR; }
	cudaDeviceProp prop;
	if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
	if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return XZB_PROG_ERROR; }
	for (auto &e : ctx->ev) cudaEventCreate(&e);
	for (auto &e : ctx->ev_mf) cudaEventCreate(&e);
	{
		// the match finder's segment kernels must get SMs while the parser kernel is resident
		int lo = 0, hi = 0;
		cudaDeviceGetStreamPriorityRange(&lo, &hi);
		if (cudaStreamCreateWithPriority(&ctx->stream_mf, cudaStreamNonBlocking, hi) != cudaSuccess) { delete ctx; return XZB_PROG_ERROR; }
		const char *ov = getenv("XZB_OVERLAP");
		ctx->overlap = !(ov && atoi(ov) == 0);
		// tools that inject into the process (ncu, compute-sanitizer) run kernels one at a time:
		// a parser waiting for a later match-finder kernel would only be rescued by its watchdog
		if (getenv("CUDA_INJECTION64_PATH") || getenv("NV_COMPUTE_PROFILER_PERFWORKS_DIR") || getenv("NV_SANITIZER_INJECTION_PORT_BASE"))
			ctx->overlap = false;
		const char *av = getenv("XZB_MF_AVOID_PARSER_SMS");
		if (av) ctx->avoid_parser_sms = atoi(av) != 0;
		const char *sm = getenv("XZB_MF_STALL_MS");
		if (sm) ctx->mf_stall_ns = (uint64_t)std::max(100, atoi(sm)) * 1000000ull;
		const char *ss = getenv("XZB_SEG_SHIFT");
		if (ss) ctx->seg_shift = (uint32_t)std::min(20, std::max(8, atoi(ss)));
	}
	xzb_make_tables(&ctx->h_tab);
	{
		cudaFuncSetAttribute(xzb_k_parse_fast<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FS<true>));
		ctx->trace_path = getenv("XZB_TRACE");
		const char *mw = getenv("XZB_MAX_WAVE_BLOCKS");
		ctx->max_wave_blocks = mw ? (uint32_t)atoi(mw) : 0;
		cudaFuncSetAttribute(xzb_k_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(XzbDec));
		if (cudaFuncSetAttribute(xzb_k_parse_dp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DS)) != cudaSuccess
				|| cudaFuncSetAttribute(xzb_k_parse_fast<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)XZB_SOLO_SMEM) != cudaSuccess) {
			fprintf(stderr, "xzb200: cannot reserve %zu B of shared memory for the parser kernel\n", sizeof(DS));
			delete ctx; return XZB_PROG_ERROR;
		}
	}
	uint64_t wide[256];
	for (int i = 0; i < 256; ++i) wide[i] = ctx->h_tab.crc32[i];
	bool ok = cudaMalloc(&ctx->d_crc32, sizeof(ctx->h_tab.crc32)) == cudaSuccess
		&& cudaMalloc(&ctx->d_crc64, sizeof(ctx->h_tab.crc64)) == cudaSuccess
		&& cudaMalloc(&ctx->d_crc32w, sizeof(wide)) == cudaSuccess
		&& cudaMalloc(&ctx->d_prices, sizeof(ctx->h_tab.prices)) == cudaSuccess;
	ok = ok && cudaMemcpy(ctx->d_crc32, ctx->h_tab.crc32, sizeof(ctx->h_tab.crc32), cudaMemcpyHostToDevice) == cudaSuccess
		&& cudaMemcpy(ctx->d_crc64, ctx->h_tab.crc64, sizeof(ctx->h_tab.crc64), cudaMemcpyHostToDevice) == cudaSuccess
		&& cudaMemcpy(ctx->d_crc32w, wide, sizeof(wide), cudaMemcpyHostToDevice) == cudaSuccess
		&& cudaMemcpy(ctx->d_prices, ctx->h_tab.prices, sizeof(ctx->h_tab.prices), cudaMemcpyHostToDevice) == cudaSuccess;
	if (!ok) { fprintf(stderr, "xzb200: CUDA init failed: %s\n", cudaGetErrorString(cudaGetLastError())); delete ctx; return XZB_PROG_ERROR; }
	*out = ctx;
	return XZB_OK;
}

extern "C" void xzb_ctx_destroy(xzb_ctx *ctx)
{
	if (!ctx) return;
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	DevBuf *bufs[] = { &ctx->keys_a, &ctx->keys_b, &ctx->vals_a, &ctx->vals_b, &ctx->keys_2, &ctx->keys_3, &ctx->prev2, &ctx->prev3,
		&ctx->prevm, &ctx->son, &ctx->mh, &ctx->mp, &ctx->ovf, &ctx->cub_tmp, &ctx->run_start, &ctx->run_len, &ctx->run_start_s,
		&ctx->run_len_s, &ctx->small, &ctx->encs, &ctx->scratch, &ctx->in_stage, &ctx->decs, &ctx->dec_in, &ctx->dec_out };
	for (DevBuf *b : bufs) free_buf(*b);
	cudaFree(ctx->d_crc32); cudaFree(ctx->d_crc64); cudaFree(ctx->d_crc32w); cudaFree(ctx->d_prices);
	for (auto &e : ctx->ev) cudaEventDestroy(e);
	for (auto &e : ctx->ev_mf) cudaEventDestroy(e);
	if (ctx->stream_mf) { cudaStreamSynchronize(ctx->stream_mf); cudaStreamDestroy(ctx->stream_mf); }
	free_buf(ctx->seg_meta);
	free_buf(ctx->trace);
	free_buf(ctx->filt_a); free_buf(ctx->filt_b); free_buf(ctx->filt_jobs);
	free_buf(ctx->out_stage); free_buf(ctx->pack_jobs);
	cudaStreamDestroy(ctx->stream);
	delete ctx;
}

extern "C" int xzb_get_stats(const xzb_ctx *ctx, xzb_stats *out) { *out = ctx->stats; return XZB_OK; }
// The filters in front of LZMA2 for the following encode calls (n = 0: none).  Validation as the reference's
// lzma_raw_encoder / validate_chain (common/filter_common.c:122-249): at most 3 + LZMA2, known IDs, Delta distance
// 1..256 (delta_common.c:46-66), BCJ start offset a multiple of the filter's alignment (simple_coder.c:276-278).
extern "C" int xzb_ctx_set_filters(xzb_ctx *ctx, const xzb_filter_spec *filters, uint32_t n)
{
	if (n > 3 || (n != 0 && filters == nullptr)) return set_err(ctx, XZB_OPTIONS_ERROR, "at most three filters before LZMA2");
	std::vector<XzbPreFilter> pre;
	for (uint32_t i = 0; i < n; ++i) {
		const uint32_t id = filters[i].id, arg = filters[i].arg;
		if (!xzb_filter_known(id)) return set_err(ctx, XZB_OPTIONS_ERROR, "filter 0x%x is not supported", id);
		if (id == XZB_FILTER_DELTA) { if (arg < 1 || arg > 256) return set_err(ctx, XZB_OPTIONS_ERROR, "delta distance %u", arg); }
		else if (arg & (xzb_filter_alignment(id) - 1)) return set_err(ctx, XZB_OPTIONS_ERROR, "BCJ start offset %u is not aligned", arg);
		pre.push_back(XzbPreFilter{ id, arg });
	}
	ctx->pre.swap(pre);
	return XZB_OK;
}

extern "C" const char *xzb_last_error(const xzb_ctx *ctx) { return ctx->err; }
extern "C" int xzb_decode_buf_reason(const xzb_ctx *ctx) { return ctx->dec_buf_reason; }

extern "C" int xzb_device_alloc(xzb_ctx *ctx, void **ptr, uint64_t size) { cudaSetDevice(ctx->device); CK(cudaMalloc(ptr, size ? size : 1)); return XZB_OK; }
extern "C" void xzb_device_free(xzb_ctx *ctx, void *ptr) { cudaSetDevice(ctx->device); cudaFree(ptr); }
extern "C" int xzb_memcpy_h2d(xzb_ctx *ctx, void *d, const void *h, uint64_t size)
{
	cudaSetDevice(ctx->device);
	CK(cudaMemcpyAsync(d, h, size, cudaMemcpyHostToDevice, ctx->stream));
	CK(cudaStreamSynchronize(ctx->stream));
	return XZB_OK;
}
extern "C" int xzb_memcpy_d2h(xzb_ctx *ctx, void *h, const void *d, uint64_t size)
{
	cudaSetDevice(ctx->device);
	CK(cudaMemcpyAsync(h, d, size, cudaMemcpyDeviceToHost, ctx->stream));
	CK(cudaStreamSynchronize(ctx->stream));
	return XZB_OK;
}

extern "C" uint32_t xzb_stream_header_encode(uint8_t out[12], uint32_t check)
{
	XzbHostTables t; xzb_make_tables(&t);
	return xzb_stream_header(t.crc32, out, check);
}
extern "C" uint32_t xzb_stream_footer_encode(uint8_t out[12], uint32_t check, uint64_t index_size)
{
	XzbHostTables t; xzb_make_tables(&t);
	return xzb_stream_footer(t.crc32, out, check, index_size);
}
extern "C" uint64_t xzb_index_encode(const xzb_index_record *records, uint64_t count, uint8_t *out)
{
	XzbHostTables t; xzb_make_tables(&t);
	std::vector<uint64_t> unp(count), unc(count);
	for (uint64_t i = 0; i < count; ++i) { unp[i] = records[i].unpadded_size; unc[i] = records[i].uncompressed_size; }
	return xzbi_index_encode(t.crc32, unp.data(), unc.data(), count, out);
}

// ------------------------------------------------------------------------------------
// Encode: one wave of B blocks
// ------------------------------------------------------------------------------------
static uint32_t bit_length(uint32_t v) { uint32_t n = 0; while (v) { ++n; v >>= 1; } return n; }

// bytes of workspace per block of size bs (upper bound), used to size waves
static uint64_t wave_bytes_per_block(uint64_t bs, const XzbParams &P)
{
	return bs * (uint64_t)(16 + 8 + 12 + 8 + 4 + 8 * P.mstride + 8) + xzb_scratch_cap(bs) + 4096;
}

static float ev_ms(cudaEvent_t a, cudaEvent_t b) { float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }

// One Block of a wave: its input is d_in[in_off .. in_off + n), `room` bytes of it readable; its framing and scratch.
struct XzbWaveBlock {
	uint64_t in_off;
	uint32_t n, room;
	uint32_t header_size, oneshot;  // see XzbEncJob
	uint64_t fit_limit;
	uint32_t scap;                  // scratch capacity
};

// Encodes the Blocks `wb` side by side.  results[b] is Block b's outcome; its finished bytes are at
// ctx->scratch + scratch_off[b].  d_in[0 .. in_bytes) covers every Block's input (the filters copy that span).
static int encode_wave(xzb_ctx *ctx, const uint8_t *d_in, uint64_t in_bytes, const std::vector<XzbWaveBlock> &wb, const XzbParams &P,
		uint32_t check, std::vector<XzbBlockResult> &results, std::vector<size_t> &scratch_off)
{
	cudaStream_t st = ctx->stream;
	const uint32_t B = (uint32_t)wb.size();
	std::vector<uint32_t> h_n(B), h_off(B);
	uint32_t bs = 0;  // the largest Block
	size_t scratch_bytes = 0;
	scratch_off.resize(B);
	for (uint32_t b = 0; b < B; ++b) {
		h_n[b] = wb[b].n; bs = std::max(bs, wb[b].n);
		scratch_off[b] = scratch_bytes; scratch_bytes += wb[b].scap;
	}
	const uint64_t N64 = xzb_wave_offsets(h_n.data(), B, h_off.data());
	const size_t N = (size_t)N64;
	const uint32_t ntiles = (uint32_t)(N / XZB_WAVE_ALIGN);
	const uint32_t hbm = bit_length(P.hash_mask);
	const uint32_t kbits_m = bit_length(B << hbm), kbits_2 = bit_length(B << 10), kbits_3 = bit_length(B << 16);
	if (N64 >= 0xFFFFFFF0ull || (uint64_t)B << hbm >= (1ull << 32) || kbits_m > 32) return set_err(ctx, XZB_PROG_ERROR, "wave too large");

	EN(ctx->keys_a, 4 * N); EN(ctx->keys_b, 4 * N); EN(ctx->vals_a, 4 * N); EN(ctx->vals_b, 4 * N);
	if (P.hash_bytes >= 3) { EN(ctx->keys_2, 4 * N); EN(ctx->prev2, 4 * N); }
	if (P.hash_bytes >= 4) { EN(ctx->keys_3, 4 * N); EN(ctx->prev3, 4 * N); }
	if (P.is_bt) EN(ctx->son, 8 * N + 64); else EN(ctx->prevm, 4 * N);
	EN(ctx->mh, 4 * N); EN(ctx->mp, 8 * (size_t)P.mstride * N); EN(ctx->ovf, 8 * N + 4096);
	EN(ctx->scratch, scratch_bytes);
	size_t tmp_sort = 0, tmp_sel = 0, tmp_sort2 = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (int64_t)N, 0, 32, st);
	if (P.is_bt) {
		XzbRunStartOp op{ nullptr, nullptr, 0, 0 };
		cub::DeviceSelect::If(nullptr, tmp_sel, cub::CountingInputIterator<uint32_t>(0), (uint32_t *)nullptr, (uint32_t *)nullptr, (int64_t)N, op, st);
		cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp_sort2, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (int64_t)N, 0, 32, st);
		EN(ctx->run_start, 4 * N); EN(ctx->run_len, 4 * N); EN(ctx->run_start_s, 4 * N); EN(ctx->run_len_s, 4 * N);
	}
	EN(ctx->cub_tmp, std::max(tmp_sort, std::max(tmp_sel, tmp_sort2)) + 256);

	// Filters in front of LZMA2 (common/filter_encoder.c:59-182): every Block's bytes go through them in chain order, on
	// a copy; match finder and parser see the result, the integrity check and the incompressible-Block fallback the input.
	const uint8_t *d_work = d_in;
	if (!ctx->pre.empty()) {
		EN(ctx->filt_a, in_bytes + 64); EN(ctx->filt_b, in_bytes + 64);
		EN(ctx->filt_jobs, sizeof(XzbFiltJob) * (size_t)B * ctx->pre.size());
		uint8_t *bufs[2] = { (uint8_t *)ctx->filt_a.p, (uint8_t *)ctx->filt_b.p };
		int which = 0;
		bool owned = false;
		std::vector<XzbFiltJob> fj((size_t)B * ctx->pre.size());
		for (size_t s = 0; s < ctx->pre.size(); ++s) {
			const XzbPreFilter f = ctx->pre[s];
			const uint8_t *src = d_work;
			uint8_t *dst;
			if (f.id == XZB_FILTER_DELTA) { dst = bufs[which]; which ^= 1; }   // out of place
			else if (!owned) { dst = bufs[which]; which ^= 1; CK(cudaMemcpyAsync(dst, d_work, in_bytes, cudaMemcpyDeviceToDevice, st)); src = dst; }
			else { dst = const_cast<uint8_t *>(d_work); }
			for (uint32_t b = 0; b < B; ++b)
				fj[s * B + b] = XzbFiltJob{ src + wb[b].in_off, dst + wb[b].in_off, wb[b].n, f.id, f.arg, 0 };
			d_work = dst; owned = true;
		}
		CK(cudaMemcpyAsync(ctx->filt_jobs.p, fj.data(), sizeof(XzbFiltJob) * fj.size(), cudaMemcpyHostToDevice, st));
		CK(cudaStreamSynchronize(st));   // fj is a local
		for (size_t s = 0; s < ctx->pre.size(); ++s) {
			xzb_k_filter<<<B, 256, 0, st>>>((const XzbFiltJob *)ctx->filt_jobs.p + s * B, 1);
			++ctx->stats.gpu_launches;
		}
	}

	// small per-wave arrays in one allocation
	const size_t off_woff = 0;  // off[B]: where each Block's positions start
	const size_t off_blocks = off_woff + ((4 * (size_t)B + 255) & ~(size_t)255);
	const size_t off_jobs = off_blocks + ((sizeof(XzbMfBlock) * B + 255) & ~(size_t)255);
	const size_t off_crcjobs = off_jobs + ((sizeof(XzbEncJob) * B + 255) & ~(size_t)255);
	const size_t off_results = off_crcjobs + ((sizeof(XzbCrcJob) * B + 255) & ~(size_t)255);
	const size_t off_pend = off_results + ((sizeof(XzbBlockResult) * B + 255) & ~(size_t)255);
	const size_t off_crcv = off_pend + ((4 * (size_t)B + 255) & ~(size_t)255);
	const size_t off_ovftop = off_crcv + ((32 * (size_t)B + 255) & ~(size_t)255);  // Check field bytes, 32 per block
	const size_t off_misc = off_ovftop + ((4 * (size_t)B + 255) & ~(size_t)255);  // [0] num_runs, [1] work counter, [2] err
	const size_t off_tiles = off_misc + 256;  // tile_block[ntiles]
	const size_t small_size = off_tiles + 4 * (size_t)ntiles + 256;
	EN(ctx->small, small_size);
	uint8_t *sm = (uint8_t *)ctx->small.p;
	std::vector<uint8_t> h_small(small_size, 0);
	uint32_t *h_woff = (uint32_t *)(h_small.data() + off_woff);
	XzbMfBlock *h_blocks = (XzbMfBlock *)(h_small.data() + off_blocks);
	XzbEncJob *h_jobs = (XzbEncJob *)(h_small.data() + off_jobs);
	XzbCrcJob *h_crcjobs = (XzbCrcJob *)(h_small.data() + off_crcjobs);
	uint32_t *h_tiles = (uint32_t *)(h_small.data() + off_tiles);
	uint64_t n_valid = 0, n_pos = 0;
	for (uint32_t b = 0; b < B; ++b) {
		const size_t off = h_off[b];
		const uint32_t n = wb[b].n;
		h_woff[b] = h_off[b];
		for (uint32_t t = h_off[b] / XZB_WAVE_ALIGN; t < (h_off[b] + xzb_wave_pad(n)) / XZB_WAVE_ALIGN; ++t) h_tiles[t] = b;
		n_pos += n;
		n_valid += n >= P.hash_bytes ? n - P.hash_bytes + 1 : 0;
		XzbMfBlock &mb = h_blocks[b];
		mb.buf = d_work + wb[b].in_off; mb.n = n;
		mb.room = wb[b].room;
		mb.prev2 = (const uint32_t *)ctx->prev2.p + off; mb.prev3 = (const uint32_t *)ctx->prev3.p + off;
		mb.prevm = (const uint32_t *)ctx->prevm.p + off;
		mb.son = (uint32_t *)ctx->son.p + 2 * off;
		mb.mh = (uint32_t *)ctx->mh.p + off;
		mb.mp = (xzb_pair *)ctx->mp.p + off * P.mstride;
		mb.ovf = (xzb_pair *)ctx->ovf.p + off;
		mb.ovf_top = (uint32_t *)(sm + off_ovftop) + b;
		mb.ovf_cap = n;
		mb.err = (uint32_t *)(sm + off_misc) + 2;
		h_jobs[b].in = d_in + wb[b].in_off; h_jobs[b].in_size = n;
		h_jobs[b].out = (uint8_t *)ctx->scratch.p + scratch_off[b]; h_jobs[b].out_cap = wb[b].scap;
		h_jobs[b].header_size = wb[b].header_size; h_jobs[b].oneshot = wb[b].oneshot; h_jobs[b].fit_limit = wb[b].fit_limit;
		h_crcjobs[b].data = d_in + wb[b].in_off; h_crcjobs[b].size = n;
	}
	CK(cudaMemcpyAsync(sm, h_small.data(), small_size, cudaMemcpyHostToDevice, st));
	const uint32_t *d_woff = (const uint32_t *)(sm + off_woff);
	const uint32_t *d_tiles = (const uint32_t *)(sm + off_tiles);
	const XzbMfBlock *d_blocks = (const XzbMfBlock *)(sm + off_blocks);
	const XzbEncJob *d_jobs = (const XzbEncJob *)(sm + off_jobs);
	const XzbCrcJob *d_crcjobs = (const XzbCrcJob *)(sm + off_crcjobs);
	XzbBlockResult *d_results = (XzbBlockResult *)(sm + off_results);
	uint32_t *d_pend = (uint32_t *)(sm + off_pend);
	uint64_t *d_crcv = (uint64_t *)(sm + off_crcv);
	uint32_t *d_misc = (uint32_t *)(sm + off_misc);

	uint32_t *keys_a = (uint32_t *)ctx->keys_a.p, *keys_b = (uint32_t *)ctx->keys_b.p;
	uint32_t *vals_a = (uint32_t *)ctx->vals_a.p, *vals_b = (uint32_t *)ctx->vals_b.p;
	uint64_t launches = 0;

	CK(cudaEventRecord(ctx->ev[0], st));
	xzb_k_hash_keys<<<ntiles, 256, 0, st>>>(d_blocks, d_tiles, d_woff, B, P, ctx->d_crc32, hbm, keys_a, (uint32_t *)ctx->keys_2.p,
			(uint32_t *)ctx->keys_3.p, vals_a, (uint32_t *)ctx->mh.p);
	++launches;
	const uint32_t pgrid = (uint32_t)((N + 255) / 256);
	size_t tb = ctx->cub_tmp.cap;
	if (P.hash_bytes >= 3) {
		CK(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp.p, tb, (const uint32_t *)ctx->keys_2.p, keys_b, vals_a, vals_b, (int64_t)N, 0, (int)kbits_2, st));
		xzb_k_prev<<<pgrid, 256, 0, st>>>(keys_b, vals_b, N, 10, B, d_woff, (uint32_t *)ctx->prev2.p);
		launches += 4;
	}
	if (P.hash_bytes >= 4) {
		tb = ctx->cub_tmp.cap;
		CK(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp.p, tb, (const uint32_t *)ctx->keys_3.p, keys_b, vals_a, vals_b, (int64_t)N, 0, (int)kbits_3, st));
		xzb_k_prev<<<pgrid, 256, 0, st>>>(keys_b, vals_b, N, 16, B, d_woff, (uint32_t *)ctx->prev3.p);
		launches += 5;
	}
	tb = ctx->cub_tmp.cap;
	CK(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp.p, tb, (const uint32_t *)keys_a, keys_b, (const uint32_t *)vals_a, vals_b, (int64_t)N, 0, (int)kbits_m, st));
	launches += 5;
	uint32_t num_runs = 0;
	// Segments of the binary-tree search (see xzb_k_bt) and the progress flag the parser polls.
	uint32_t seg_shift = ctx->seg_shift;
	while ((((uint64_t)bs + (1u << seg_shift) - 1) >> seg_shift) > (1u << (32 - XZB_RUN_LEN_BITS))) ++seg_shift;  // segment index must fit the run key
	const uint32_t nseg = P.is_bt ? (uint32_t)(((uint64_t)bs + (1u << seg_shift) - 1) >> seg_shift) : 1;
	const size_t seg_meta_words = 2 * (size_t)nseg + 8 + 256;
	EN(ctx->seg_meta, 4 * seg_meta_words);
	uint32_t *d_flag = (uint32_t *)ctx->seg_meta.p, *d_seg_first = d_flag + 1, *d_seg_counters = d_seg_first + nseg + 1;
	uint32_t *d_parser_sm = d_seg_counters + nseg + 2;  // parser_sm[256]: "a parser CTA runs on this SM"
	CK(cudaMemsetAsync(ctx->seg_meta.p, P.is_bt ? 0x00 : 0xFF, 4 * seg_meta_words, st));  // hash chains: everything is ready before the parser starts
	// The parser may run beside the match finder when every parser CTA is resident at once (one per SM):
	// otherwise queued parser CTAs could keep the later segment kernels from being scheduled.
	const bool overlap = ctx->overlap && P.is_bt && B <= (uint32_t)ctx->sm_count;
	cudaStream_t st_mf = overlap ? ctx->stream_mf : st;
	if (!P.is_bt) {
		xzb_k_prev<<<pgrid, 256, 0, st>>>(keys_b, vals_b, N, hbm, B, d_woff, (uint32_t *)ctx->prevm.p);
		++launches;
	} else {
		XzbRunStartOp op{ keys_b, vals_b, B << hbm, seg_shift };
		tb = ctx->cub_tmp.cap;
		CK(cub::DeviceSelect::If(ctx->cub_tmp.p, tb, cub::CountingInputIterator<uint32_t>(0), (uint32_t *)ctx->run_start.p, d_misc, (int64_t)N, op, st));
		xzb_k_run_key<<<pgrid, 256, 0, st>>>((const uint32_t *)ctx->run_start.p, d_misc, (uint32_t)n_valid, vals_b, seg_shift, nseg, (uint32_t *)ctx->run_len.p);
		CK(cudaMemcpyAsync(&num_runs, d_misc, 4, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		launches += 4;
		if (num_runs > 0) {
			tb = ctx->cub_tmp.cap;
			CK(cub::DeviceRadixSort::SortPairsDescending(ctx->cub_tmp.p, tb, (const uint32_t *)ctx->run_len.p, (uint32_t *)ctx->run_len_s.p,
					(const uint32_t *)ctx->run_start.p, (uint32_t *)ctx->run_start_s.p, (int64_t)num_runs, 0, 32, st));
			launches += 5;
		}
		xzb_k_seg_bounds<<<(num_runs + 255) / 256 + 1, 256, 0, st>>>((const uint32_t *)ctx->run_len_s.p, d_misc, nseg, d_seg_first);
		++launches;
	}
	CK(cudaEventRecord(ctx->ev[1], st));
	auto launch_crc = [&]() {
		if (check == 1 || check == 4) {
			const bool c64 = check == 4;
			xzb_k_crc<<<B, 1024, 0, st>>>(d_crcjobs, c64 ? ctx->d_crc64 : ctx->d_crc32w, c64 ? ~0ull : 0xFFFFFFFFull, d_crcv, 4, nullptr);
			++launches;
		}
	};
	uint32_t *d_trace = nullptr;
	const uint32_t trace_cap = ctx->trace_path ? (uint32_t)std::min<uint64_t>(in_bytes, 1u << 25) : 0;
	if (ctx->trace_path) {
		EN(ctx->trace, 4 * (3 * (size_t)trace_cap + 4));
		CK(cudaMemsetAsync(ctx->trace.p, 0, 16, st));
		d_trace = (uint32_t *)ctx->trace.p + 1;
	}
	auto launch_parse = [&]() {
		if (P.mode == XZB_MODE_NORMAL) {
			xzb_k_parse_dp<<<B, P.nice_len > 127 ? 224 : 512, sizeof(DS), st>>>(d_jobs, d_blocks, P, ctx->d_prices, d_flag, d_parser_sm, ctx->mf_stall_ns, d_results, d_pend,
					d_trace, trace_cap);
		} else if (B > (uint32_t)ctx->sm_count) {
			// Fast mode has two forms.  With more Blocks in the wave than SMs the coder-warp form runs at its own size, so
			// several Blocks share an SM (measured 24 % slower per Block on 8 x 4 MiB `T` at -1, but several times the
			// Blocks in flight); a wave that leaves SMs idle anyway runs the two-warp form, one Block per SM.
			xzb_k_parse_fast<true><<<B, 96, sizeof(FS<true>), st>>>(d_jobs, d_blocks, P, d_flag, d_parser_sm, ctx->mf_stall_ns, d_results, d_pend);
		} else {
			xzb_k_parse_fast<false><<<B, 96, XZB_SOLO_SMEM, st>>>(d_jobs, d_blocks, P, d_flag, d_parser_sm, ctx->mf_stall_ns, d_results, d_pend);
		}
		++launches;
	};
	if (!P.is_bt) {
		xzb_k_hc<<<2 * ntiles, 128, 0, st>>>(d_blocks, d_tiles, d_woff, P);
		++launches;
		CK(cudaEventRecord(ctx->ev[2], st));
		if (check == 10) { xzb_k_sha256<<<B, 32, 0, st>>>(d_crcjobs, (uint8_t *)d_crcv, nullptr); ++launches; }
	} else {
		// Beside the parser the search keeps off the parser's SMs (see xzb_k_bt): the launch is
		// oversubscribed by the CTAs that will retire there, `live` CTAs do the work.
		const bool avoid = overlap && ctx->avoid_parser_sms && (uint32_t)ctx->sm_count >= B + 16;
		const uint32_t mf_sms = avoid ? (uint32_t)ctx->sm_count - B : (uint32_t)ctx->sm_count;
		if (overlap) CK(cudaStreamWaitEvent(st_mf, ctx->ev[1], 0));
		CK(cudaEventRecord(ctx->ev_mf[0], st_mf));
		int per_sm = 0;
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, xzb_k_bt, 128, 0));
		if (per_sm < 1) per_sm = 1;
		const uint32_t live = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)mf_sms * per_sm, (num_runs / nseg + 127) / 128 + 1));
		const uint32_t grid = avoid ? live + B * (uint32_t)per_sm : live;
		for (uint32_t sg = 0; sg < nseg; ++sg) {
			if (num_runs > 0) {
				xzb_k_bt<<<grid, 128, 0, st_mf>>>(d_blocks, P, keys_b, vals_b, (const uint32_t *)ctx->run_start_s.p, (const uint32_t *)ctx->run_len_s.p,
						d_seg_first, sg, hbm, d_seg_counters, avoid ? d_parser_sm : nullptr, live);
				++launches;
			}
			xzb_k_publish<<<1, 1, 0, st_mf>>>(d_flag, sg + 1 < nseg ? (sg + 1) << seg_shift : 0xFFFFFFFFu);
			++launches;
		}
		CK(cudaEventRecord(ctx->ev_mf[1], st_mf));
		if (!overlap) CK(cudaEventRecord(ctx->ev[2], st));
		// SHA-256 needs only the input: behind the search on its stream, i.e. beside the parser when overlapping
		if (check == 10) { xzb_k_sha256<<<B, 32, 0, st_mf>>>(d_crcjobs, (uint8_t *)d_crcv, nullptr); ++launches; CK(cudaEventRecord(ctx->ev_mf[2], st_mf)); }
	}
	launch_crc();
	CK(cudaEventRecord(ctx->ev[3], st));
	results.resize(B);
	for (int attempt = 0;; ++attempt) {
		launch_parse();
		CK(cudaEventRecord(ctx->ev[4], st));
		if (P.is_bt && overlap) CK(cudaStreamWaitEvent(st, check == 10 ? ctx->ev_mf[2] : ctx->ev_mf[1], 0));  // also: workspace is reused by the next wave
		xzb_k_finalize<<<B, 256, 0, st>>>(d_jobs, ctx->d_crc32, P, check, (const uint8_t *)d_crcv, d_pend, d_results);
		++launches;
		CK(cudaEventRecord(ctx->ev[5], st));
		CK(cudaMemcpyAsync(results.data(), d_results, sizeof(XzbBlockResult) * B, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		// Watchdog path: a parser CTA saw no match-finder progress for XZB_MF_STALL_NS (kernels were not
		// running side by side after all).  Every segment is finished by now; parse again.
		bool stalled = false;
		for (uint32_t b = 0; b < B; ++b) stalled = stalled || results[b].ret == XZB_MF_STALL;
		if (!stalled) break;
		if (attempt > 0) return set_err(ctx, XZB_PROG_ERROR, "parser stalled waiting for the match finder");
		if (ctx->mf_stalls++ == 0) fprintf(stderr, "xzb200: match finder and parser kernels did not overlap; parsing again after the match finder\n");
		ctx->overlap = false;
	}
	if (d_trace != nullptr) {
		uint32_t n = 0;
		CK(cudaMemcpy(&n, ctx->trace.p, 4, cudaMemcpyDeviceToHost));
		std::vector<uint32_t> t(3 * (size_t)n + 1);
		CK(cudaMemcpy(t.data(), (uint32_t *)ctx->trace.p + 1, 12 * (size_t)n, cudaMemcpyDeviceToHost));
		if (FILE *f = fopen(ctx->trace_path, "wb")) { fwrite(t.data(), 12, n, f); fclose(f); }
	}
	uint32_t h_misc[4] = { 0, 0, 0, 0 };
	CK(cudaMemcpyAsync(h_misc, d_misc, sizeof(h_misc), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	CK(cudaGetLastError());
	if (h_misc[2] != 0) return set_err(ctx, (int)h_misc[2], "match store overflow pool exhausted");
	ctx->stats.ms_mf_prep += ev_ms(ctx->ev[0], ctx->ev[1]);
	if (P.is_bt && overlap) {  // the match finder ran beside the parser: its own stream's clock
		ctx->stats.ms_mf += ev_ms(ctx->ev_mf[0], ctx->ev_mf[1]);
		ctx->stats.ms_other += ev_ms(ctx->ev[1], ctx->ev[3]) + ev_ms(ctx->ev[4], ctx->ev[5]);
	} else {
		ctx->stats.ms_mf += ev_ms(ctx->ev[1], ctx->ev[2]);
		ctx->stats.ms_other += ev_ms(ctx->ev[2], ctx->ev[3]) + ev_ms(ctx->ev[4], ctx->ev[5]);
	}
	ctx->stats.ms_parse += ev_ms(ctx->ev[3], ctx->ev[4]);
	ctx->stats.gpu_launches += launches;
	ctx->stats.n_blocks += B;
	ctx->stats.n_positions += n_pos;
	ctx->stats.mf_bytes_algorithmic += n_valid * (uint64_t)(P.is_bt ? 33 : 29);
	for (uint32_t b = 0; b < B; ++b) {
		ctx->stats.n_symbols += results[b].n_symbols;
		ctx->stats.n_chunks_lzma += results[b].n_chunks_lzma;
		ctx->stats.n_chunks_raw += results[b].n_chunks_raw;
		ctx->stats.n_fallback_blocks += results[b].fallback;
	}
	return XZB_OK;
}

// Device memory an encode wave may take: 85 % of what is free, counting the workspace this context already holds,
// less `reserve`.
static uint64_t wave_budget(xzb_ctx *ctx, uint64_t reserve)
{
	size_t free_b = 0, total_b = 0;
	cudaMemGetInfo(&free_b, &total_b);
	uint64_t held = 0;
	const DevBuf *bufs[] = { &ctx->keys_a, &ctx->keys_b, &ctx->vals_a, &ctx->vals_b, &ctx->keys_2, &ctx->keys_3, &ctx->prev2, &ctx->prev3,
		&ctx->prevm, &ctx->son, &ctx->mh, &ctx->mp, &ctx->ovf, &ctx->cub_tmp, &ctx->run_start, &ctx->run_len, &ctx->run_start_s,
		&ctx->run_len_s, &ctx->encs, &ctx->scratch };
	for (const DevBuf *b : bufs) held += b->cap;
	const uint64_t budget = (uint64_t)((free_b + held) * 0.85);
	return budget > reserve ? budget - reserve : 0;
}

static uint32_t pick_wave_blocks(xzb_ctx *ctx, uint64_t bs, const XzbParams &P, uint64_t nblocks, uint64_t reserve)
{
	const uint64_t budget = wave_budget(ctx, reserve);
	uint64_t per = wave_bytes_per_block(bs, P) + (P.is_bt ? 16 * bs : 0);
	uint64_t w = per ? budget / per : 1;
	const uint32_t hbm = bit_length(P.hash_mask);
	const uint64_t key_cap = (1ull << (32 - hbm)) - 1;  // (B << hbm) must fit 32 bits
	w = std::min<uint64_t>(w, key_cap);
	w = std::min<uint64_t>(w, 0xFFFFFFF0ull / xzb_wave_pad(bs) - 1);
	w = std::min<uint64_t>(w, nblocks);
	if (ctx->max_wave_blocks) w = std::min<uint64_t>(w, ctx->max_wave_blocks);  // XZB_MAX_WAVE_BLOCKS (tests: force several waves)
	return (uint32_t)std::max<uint64_t>(w, 1);
}

// Starts an encode call: clears the call's stats and error, derives the coder parameters from the options and the
// context's filter chain, and checks the Check ID.
static int encode_begin(xzb_ctx *ctx, const xzb_lzma_options *opt, uint32_t check, XzbParams &P)
{
	cudaSetDevice(ctx->device);
	memset(&ctx->stats, 0, sizeof(ctx->stats));
	ctx->err[0] = 0;
	const int r = xzb_make_params((const XzbLzmaOptions *)opt, &P);
	if (r != XZB_OK) return set_err(ctx, r, "unsupported LZMA2 options");
	if (!ctx->pre.empty()) {
		// Filter Flags of the filters in front of LZMA2: ID, size of properties, properties (filter_flags_encoder.c:31-56;
		// delta_encoder.c:119-131: distance - 1; simple_encoder.c:15-28: nothing, or the start offset as 4 bytes)
		for (const XzbPreFilter &f : ctx->pre) {
			P.ff[P.ff_len++] = (uint8_t)f.id;
			if (f.id == XZB_FILTER_DELTA) { P.ff[P.ff_len++] = 1; P.ff[P.ff_len++] = (uint8_t)(f.arg - 1); }
			else if (f.arg == 0) P.ff[P.ff_len++] = 0;
			else { P.ff[P.ff_len++] = 4; for (int i = 0; i < 4; ++i) P.ff[P.ff_len++] = (uint8_t)(f.arg >> (8 * i)); }
		}
		P.n_pre = (uint8_t)ctx->pre.size();
	}
	if (xzb_check_size(check) == 0xFFFFFFFFu) return set_err(ctx, XZB_UNSUPPORTED_CHECK, "check %u not supported", check);
	return XZB_OK;
}

// Places finished Blocks (and, for framed jobs, whole one-shot Streams) with one xzb_k_pack_streams launch, then
// synchronises.  host_out == nullptr: every job's dst is a device address.  Otherwise each dst is an offset into a
// staging area of stage_bytes, which comes back to host_out with one copy.
static int place_blocks(xzb_ctx *ctx, std::vector<XzbPackJob> &jobs, uint32_t check, uint8_t *host_out, size_t stage_bytes)
{
	cudaStream_t st = ctx->stream;
	if (!jobs.empty()) {
		if (host_out != nullptr) {
			EN(ctx->out_stage, stage_bytes + 64);
			for (XzbPackJob &j : jobs) j.dst = (uint8_t *)ctx->out_stage.p + (size_t)j.dst;
		}
		EN(ctx->pack_jobs, sizeof(XzbPackJob) * jobs.size());
		CK(cudaMemcpyAsync(ctx->pack_jobs.p, jobs.data(), sizeof(XzbPackJob) * jobs.size(), cudaMemcpyHostToDevice, st));
		xzb_k_pack_streams<<<(uint32_t)jobs.size(), 256, 0, st>>>((const XzbPackJob *)ctx->pack_jobs.p, ctx->d_crc32, check);
		++ctx->stats.gpu_launches;
		if (host_out != nullptr && stage_bytes > 0) CK(cudaMemcpyAsync(host_out, ctx->out_stage.p, stage_bytes, cudaMemcpyDeviceToHost, st));
	}
	CK(cudaStreamSynchronize(st));   // also: `jobs` is the source of the copy above
	CK(cudaGetLastError());
	return XZB_OK;
}

static int encode_common(xzb_ctx *ctx, const uint8_t *in, bool in_is_device, uint64_t in_size, const xzb_lzma_options *opt, uint32_t check,
		uint64_t block_size, uint8_t *out, bool out_is_device, uint64_t out_cap, uint64_t *out_size, xzb_index_record *records,
		bool whole_stream)
{
	XzbParams P;
	int r = encode_begin(ctx, opt, check, P);
	if (r != XZB_OK) return r;
	if (block_size == 0) block_size = std::max<uint64_t>((uint64_t)P.dict_size * 3, 1u << 20);  // lzma_lzma2_block_size, lzma2_encoder.c:403-413
	if (block_size > (1ull << 30)) return set_err(ctx, XZB_OPTIONS_ERROR, "block_size > 1 GiB is not supported on the GPU path");
	const uint64_t nblocks = (in_size + block_size - 1) / block_size;
	const uint32_t bs = (uint32_t)block_size;
	std::vector<xzb_index_record> recs(nblocks);
	uint64_t pos = 0;
	cudaStream_t st = ctx->stream;
	CK(cudaEventRecord(ctx->ev[6], st));
	if (whole_stream) {
		uint8_t hdr[12];
		xzb_stream_header(ctx->h_tab.crc32, hdr, check);
		if (out_cap < 12) return set_err(ctx, XZB_BUF_ERROR, "output too small");
		if (out_is_device) CK(cudaMemcpyAsync(out, hdr, 12, cudaMemcpyHostToDevice, st)); else memcpy(out, hdr, 12);
		pos = 12;
	}
	uint64_t done = 0;
	const uint64_t bound = xzbi_block_bound(block_size);
	const uint32_t header_size = xzb_block_header_size(bound, block_size, P.ff_len);
	while (done < nblocks) {
		const uint64_t stage = (uint64_t)bs * std::min<uint64_t>(nblocks - done, 256);
		const uint32_t W = pick_wave_blocks(ctx, bs, P, nblocks - done, (in_is_device ? 0 : stage) + (out_is_device ? 0 : stage));
		const uint64_t off = done * block_size;
		const uint64_t wave_bytes = std::min<uint64_t>((uint64_t)W * bs, in_size - off);
		const uint8_t *d_wave;
		if (in_is_device) {
			d_wave = in + off;
		} else {
			EN(ctx->in_stage, (size_t)W * bs + 64);
			CK(cudaEventRecord(ctx->ev[8], st));
			CK(cudaMemcpyAsync(ctx->in_stage.p, in + off, wave_bytes, cudaMemcpyHostToDevice, st));
			CK(cudaEventRecord(ctx->ev[9], st));
			d_wave = (const uint8_t *)ctx->in_stage.p;
		}
		const bool has_slack = !in_is_device || off + wave_bytes < in_size;
		std::vector<XzbWaveBlock> wb(W);
		for (uint32_t b = 0; b < W; ++b) {
			const uint32_t n = (uint32_t)std::min<uint64_t>(bs, wave_bytes - (uint64_t)b * bs);
			wb[b] = XzbWaveBlock{ (uint64_t)b * bs, n, (b + 1 < W || has_slack) ? n + 8 : n, header_size, 0, bound, xzb_scratch_cap(block_size) };
		}
		std::vector<XzbBlockResult> results;
		std::vector<size_t> sc_off;
		r = encode_wave(ctx, d_wave, wave_bytes, wb, P, check, results, sc_off);
		if (r != XZB_OK) return r;
		if (!in_is_device) ctx->stats.ms_h2d += ev_ms(ctx->ev[8], ctx->ev[9]);
		CK(cudaEventRecord(ctx->ev[10], st));
		const uint64_t pos0 = pos;
		std::vector<XzbPackJob> jobs(W);
		for (uint32_t b = 0; b < W; ++b) {
			const XzbBlockResult &res = results[b];
			if (res.ret != XZB_OK) return set_err(ctx, (int)res.ret, "block %llu failed", (unsigned long long)(done + b));
			if (pos + res.total_size > out_cap) return set_err(ctx, XZB_BUF_ERROR, "output buffer too small");
			uint8_t *dst = out_is_device ? out + pos : (uint8_t *)(uintptr_t)(pos - pos0);
			jobs[b] = XzbPackJob{ (const uint8_t *)ctx->scratch.p + sc_off[b], dst, 0, 0, res.total_size, 0 };
			pos += res.total_size;
			recs[done + b].unpadded_size = res.unpadded_size;
			recs[done + b].uncompressed_size = wb[b].n;
		}
		r = place_blocks(ctx, jobs, check, out_is_device ? nullptr : out + pos0, pos - pos0);
		if (r != XZB_OK) return r;
		CK(cudaEventRecord(ctx->ev[11], st));
		CK(cudaStreamSynchronize(st));
		if (!out_is_device) ctx->stats.ms_d2h += ev_ms(ctx->ev[10], ctx->ev[11]); else ctx->stats.ms_other += ev_ms(ctx->ev[10], ctx->ev[11]);
		done += W;
	}
	if (whole_stream) {
		const uint64_t isz = xzb_index_encode(recs.data(), nblocks, nullptr);
		if (pos + isz + 12 > out_cap) return set_err(ctx, XZB_BUF_ERROR, "output buffer too small");
		std::vector<uint8_t> tail(isz + 12);
		xzb_index_encode(recs.data(), nblocks, tail.data());
		xzb_stream_footer(ctx->h_tab.crc32, tail.data() + isz, check, isz);
		if (out_is_device) CK(cudaMemcpyAsync(out + pos, tail.data(), tail.size(), cudaMemcpyHostToDevice, st)); else memcpy(out + pos, tail.data(), tail.size());
		pos += tail.size();
	}
	CK(cudaEventRecord(ctx->ev[7], st));
	CK(cudaStreamSynchronize(st));
	ctx->stats.ms_total = ev_ms(ctx->ev[6], ctx->ev[7]);
	if (records) for (uint64_t i = 0; i < nblocks; ++i) records[i] = recs[i];
	*out_size = pos;
	return XZB_OK;
}

extern "C" int xzb_encode_blocks_device(xzb_ctx *ctx, const void *d_in, uint64_t in_size, const xzb_lzma_options *opt, uint32_t check,
		uint64_t block_size, void *d_out, uint64_t d_out_cap, uint64_t *out_size, xzb_index_record *records)
{
	return encode_common(ctx, (const uint8_t *)d_in, true, in_size, opt, check, block_size, (uint8_t *)d_out, true, d_out_cap, out_size, records, false);
}

extern "C" int xzb_encode_blocks_host(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, const xzb_lzma_options *opt, uint32_t check,
		uint64_t block_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size, xzb_index_record *records)
{
	return encode_common(ctx, in, false, in_size, opt, check, block_size, out, false, out_cap, out_size, records, false);
}

extern "C" int xzb_stream_encode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, const xzb_lzma_options *opt, uint32_t check,
		uint64_t block_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size)
{
	return encode_common(ctx, in, false, in_size, opt, check, block_size, out, false, out_cap, out_size, nullptr, true);
}

// A Block with no uncompressed data, as lzma_block_buffer_encode() produces it for in_size == 0
// (block_buffer_encoder.c:165-325 with lzma2_bound(0) == 1): header, the LZMA2 end marker, padding, check of
// zero bytes.  Host only: there is nothing to compute.  Returns the Block's size.
extern "C" uint32_t xzb_empty_block_encode(uint8_t *out, const xzb_lzma_options *opt, uint32_t check)
{
	XzbHostTables tab;
	xzb_make_tables(&tab);
	const uint32_t hs = xzb_block_header_size(1, 0);
	xzb_block_header_encode(tab.crc32, out, hs, 1, 0, xzb_lzma2_dict_prop(opt->dict_size));
	uint32_t pos = hs;
	out[pos++] = 0x00;
	while (pos & 3) out[pos++] = 0x00;
	uint8_t cb[32] = { 0 };
	if (check == 10) xzb_sha256(out, 0, cb);
	xzb_put_check(out + pos, check, cb);
	return pos + xzb_check_size(check);
}

// lzma_stream_buffer_encode() / lzma_easy_buffer_encode() (common/stream_buffer_encoder.c:43-140,
// easy_buffer_encoder.c:16-27): Stream Header, ONE Block over the whole input with
// lzma_block_buffer_encode() framing, Index, Stream Footer.
extern "C" uint64_t xzb_stream_buffer_bound(uint64_t in_size)
{
	const uint64_t bb = xzb_block_bound(in_size);  // stream_buffer_encoder.c:17-40
	const uint64_t hb = 2 * 12 + ((1 + 1 + 2 * 9 + 4 + 3) & ~3);
	if (bb == 0 || ((~0ull) >> 1) - bb < hb) return 0;
	return bb + hb;
}

// n independent one-shot Streams.  The items are encoded in waves of similar sizes (xzb_plan_waves), each Block framed
// as lzma_block_buffer_encode() does (block_encode_normal(), block_buffer_encoder.c:165-183: header sized from
// lzma2_bound(n), the LZMA2 data alone must fit) and turned into its Stream by xzb_k_pack_streams.
static int encode_batch(xzb_ctx *ctx, uint32_t n, const uint8_t *in, bool in_is_device, const uint64_t *in_off, const uint64_t *in_size,
		const xzb_lzma_options *opt, uint32_t check, uint8_t *out, bool out_is_device, const uint64_t *out_off, const uint64_t *out_cap,
		uint64_t *out_size, uint32_t *ret)
{
	XzbParams P;
	int r = encode_begin(ctx, opt, check, P);
	if (r != XZB_OK) return r;
	cudaStream_t st = ctx->stream;
	CK(cudaEventRecord(ctx->ev[6], st));
	std::vector<uint32_t> items;       // the items with a Block
	std::vector<uint64_t> sizes;
	std::vector<XzbPackJob> empties;   // Streams with no Block
	std::vector<uint32_t> empty_items;
	for (uint32_t i = 0; i < n; ++i) {
		out_size[i] = 0; ret[i] = XZB_OK;
		if (in_size[i] > (1ull << 30)) { ret[i] = XZB_OPTIONS_ERROR; set_err(ctx, XZB_OPTIONS_ERROR, "block_size > 1 GiB is not supported on the GPU path"); }
		else if (in_size[i] == 0) { empty_items.push_back(i); }
		else { items.push_back(i); sizes.push_back(in_size[i]); }
	}
	// Host output goes through a staging area packed in call order of the items that fit, then back in one copy.
	std::vector<uint8_t> host_stage;
	auto place = [&](const std::vector<uint32_t> &who, std::vector<XzbPackJob> &jobs) -> int {
		uint64_t stage = 0;
		std::vector<XzbPackJob> keep;
		std::vector<uint32_t> kept;
		for (size_t k = 0; k < jobs.size(); ++k) {
			const uint32_t i = who[k];
			const uint64_t size = xzb_oneshot_stream_size(jobs[k].size, jobs[k].unpadded, jobs[k].uncomp);
			if (size > out_cap[i]) { ret[i] = XZB_BUF_ERROR; set_err(ctx, XZB_BUF_ERROR, "output buffer too small"); continue; }
			out_size[i] = size;
			jobs[k].dst = out_is_device ? out + out_off[i] : (uint8_t *)(uintptr_t)stage;
			stage += (size + 15) & ~15ull;
			keep.push_back(jobs[k]); kept.push_back(i);
		}
		if (!out_is_device) host_stage.resize(stage);
		const int pr = place_blocks(ctx, keep, check, out_is_device ? nullptr : host_stage.data(), stage);
		if (pr != XZB_OK) return pr;
		if (!out_is_device)
			for (size_t k = 0; k < keep.size(); ++k)
				memcpy(out + out_off[kept[k]], host_stage.data() + (keep[k].dst - (uint8_t *)ctx->out_stage.p), out_size[kept[k]]);
		return XZB_OK;
	};
	const uint32_t hbm = bit_length(P.hash_mask);
	std::vector<uint32_t> order, wave_start;
	xzb_plan_waves(sizes.data(), (uint32_t)sizes.size(), xzb_wave_cost(P), wave_budget(ctx, 0), hbm, ctx->max_wave_blocks, &order, &wave_start);
	for (size_t w = 0; w + 1 < wave_start.size(); ++w) {
		const uint32_t B = wave_start[w + 1] - wave_start[w];
		std::vector<uint32_t> who(B), wn(B), woff(B);
		for (uint32_t b = 0; b < B; ++b) { who[b] = items[order[wave_start[w] + b]]; wn[b] = (uint32_t)in_size[who[b]]; }
		// the wave's inputs side by side in HBM, each at its Block's workspace offset; the 64 bytes behind the last one
		// are the slack the match finder may read past every Block
		const uint64_t total = xzb_wave_offsets(wn.data(), B, woff.data());
		EN(ctx->in_stage, total + 64);
		uint8_t *d_wave = (uint8_t *)ctx->in_stage.p;
		CK(cudaEventRecord(ctx->ev[8], st));
		for (uint32_t b = 0; b < B; ++b)
			CK(cudaMemcpyAsync(d_wave + woff[b], in + in_off[who[b]], wn[b], in_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
		CK(cudaEventRecord(ctx->ev[9], st));
		std::vector<XzbWaveBlock> wb(B);
		for (uint32_t b = 0; b < B; ++b) {
			const uint32_t hs = xzb_block_header_size(xzb_lzma2_bound(wn[b]), wn[b], P.ff_len);
			wb[b] = XzbWaveBlock{ woff[b], wn[b], wn[b] + 8, hs, 1, hs + xzb_lzma2_bound(wn[b]), xzb_scratch_cap(wn[b]) };
		}
		std::vector<XzbBlockResult> results;
		std::vector<size_t> sc_off;
		r = encode_wave(ctx, d_wave, total, wb, P, check, results, sc_off);
		if (r != XZB_OK) return r;
		ctx->stats.ms_h2d += ev_ms(ctx->ev[8], ctx->ev[9]);
		std::vector<XzbPackJob> jobs;
		std::vector<uint32_t> placed;
		for (uint32_t b = 0; b < B; ++b) {
			const XzbBlockResult &res = results[b];
			if (res.ret != XZB_OK) { ret[who[b]] = res.ret; set_err(ctx, (int)res.ret, "item %u failed", who[b]); continue; }
			jobs.push_back(XzbPackJob{ (const uint8_t *)ctx->scratch.p + sc_off[b], nullptr, res.unpadded_size, wn[b], res.total_size, 1 });
			placed.push_back(who[b]);
		}
		r = place(placed, jobs);
		if (r != XZB_OK) return r;
	}
	for (size_t k = 0; k < empty_items.size(); ++k) empties.push_back(XzbPackJob{ nullptr, nullptr, 0, 0, 0, 1 });
	r = place(empty_items, empties);
	if (r != XZB_OK) return r;
	CK(cudaEventRecord(ctx->ev[7], st));
	CK(cudaStreamSynchronize(st));
	ctx->stats.ms_total = ev_ms(ctx->ev[6], ctx->ev[7]);
	return XZB_OK;
}

extern "C" int xzb_stream_buffer_encode_batch(xzb_ctx *ctx, uint32_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_size,
		const xzb_lzma_options *opt, uint32_t check, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint32_t *ret)
{
	return encode_batch(ctx, n, in, false, in_off, in_size, opt, check, out, false, out_off, out_cap, out_size, ret);
}

extern "C" int xzb_stream_buffer_encode_batch_device(xzb_ctx *ctx, uint32_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_size,
		const xzb_lzma_options *opt, uint32_t check, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint32_t *ret)
{
	return encode_batch(ctx, n, in, true, in_off, in_size, opt, check, out, true, out_off, out_cap, out_size, ret);
}

extern "C" int xzb_stream_buffer_encode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, const xzb_lzma_options *opt, uint32_t check,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size)
{
	const uint64_t zero = 0;
	uint64_t size = 0;
	uint32_t ret = XZB_OK;
	const int r = encode_batch(ctx, 1, in, false, &zero, &in_size, opt, check, out, false, &zero, &out_cap, &size, &ret);
	if (r != XZB_OK) return r;
	if (ret == XZB_OK) *out_size = size;
	return (int)ret;
}

// ------------------------------------------------------------------------------------
// Decode
// ------------------------------------------------------------------------------------
// Decodes the Blocks `jobs` side by side; checks[b] is the Check ID whose value crcs[b] (CRC32 / CRC64) or
// shas[32 b ..] (SHA-256, when shas is given) receives for what Block b produced; 0 or any other ID: none.
static int decode_batch(xzb_ctx *ctx, const std::vector<XzbDecJob> &jobs, const std::vector<uint32_t> &checks, std::vector<XzbDecResult> &results, std::vector<uint64_t> &crcs,
		std::vector<uint8_t> *shas = nullptr, const std::vector<XzbBlockHeader> *chains = nullptr)
{
	cudaStream_t st = ctx->stream;
	const uint32_t B = (uint32_t)jobs.size();
	results.assign(B, XzbDecResult{ 0, 0, 0, 0 });
	crcs.assign(B, 0);
	if (B == 0) return XZB_OK;
	const size_t off_jobs = 0;
	const size_t off_res = (sizeof(XzbDecJob) * B + 255) & ~(size_t)255;
	const size_t off_crcjobs = off_res + ((sizeof(XzbDecResult) * B + 255) & ~(size_t)255);
	const size_t off_crcv = off_crcjobs + ((sizeof(XzbCrcJob) * B + 255) & ~(size_t)255);
	const size_t total = off_crcv + 32 * (size_t)B + 256;
	EN(ctx->small, total);
	uint8_t *sm = (uint8_t *)ctx->small.p;
	CK(cudaMemcpyAsync(sm + off_jobs, jobs.data(), sizeof(XzbDecJob) * B, cudaMemcpyHostToDevice, st));
	CK(cudaEventRecord(ctx->ev[0], st));
	xzb_k_decode<<<B, 32, sizeof(XzbDec), st>>>((const XzbDecJob *)(sm + off_jobs), (XzbDecResult *)(sm + off_res));
	CK(cudaEventRecord(ctx->ev[1], st));
	CK(cudaMemcpyAsync(results.data(), sm + off_res, sizeof(XzbDecResult) * B, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	ctx->stats.gpu_launches += 1;
	if (chains != nullptr) {
		// Delta / BCJ behind LZMA2 (common/filter_decoder.c:44-139): undone in reverse chain order over what each Block
		// produced, before the integrity check looks at the bytes
		uint32_t depth = 0;
		for (const XzbBlockHeader &hb : *chains) depth = std::max(depth, hb.n_pre);
		for (uint32_t lvl = 0; lvl < depth; ++lvl) {
			std::vector<XzbFiltJob> fj(B);
			for (uint32_t b = 0; b < B; ++b) {
				const XzbBlockHeader &hb = (*chains)[b];
				fj[b] = XzbFiltJob{ jobs[b].out, jobs[b].out, 0, 0, 0, 0 };
				if (lvl < hb.n_pre) { const XzbPreFilter f = hb.pre[hb.n_pre - 1 - lvl]; fj[b].size = results[b].out_used; fj[b].id = f.id; fj[b].arg = f.arg; }
			}
			EN(ctx->filt_jobs, sizeof(XzbFiltJob) * (size_t)B);
			CK(cudaMemcpyAsync(ctx->filt_jobs.p, fj.data(), sizeof(XzbFiltJob) * B, cudaMemcpyHostToDevice, st));
			CK(cudaStreamSynchronize(st));
			xzb_k_filter<<<B, 256, 0, st>>>((const XzbFiltJob *)ctx->filt_jobs.p, 0);
			ctx->stats.gpu_launches += 1;
		}
	}
	// the integrity check of what each Block produced: one launch per check type over the Blocks that carry it
	if (shas != nullptr) shas->assign(32 * (size_t)B, 0);
	for (const uint32_t c : { 1u, 4u, 10u }) {
		if (c == 10 && shas == nullptr) continue;
		std::vector<XzbCrcJob> cj;
		std::vector<uint32_t> who;
		for (uint32_t b = 0; b < B; ++b)
			if (checks[b] == c) { cj.push_back(XzbCrcJob{ jobs[b].out, results[b].out_used }); who.push_back(b); }
		if (cj.empty()) continue;
		const uint32_t nc = (uint32_t)cj.size();
		CK(cudaMemcpyAsync(sm + off_crcjobs, cj.data(), sizeof(XzbCrcJob) * nc, cudaMemcpyHostToDevice, st));
		std::vector<uint8_t> got(32 * (size_t)nc);
		if (c == 10) {
			xzb_k_sha256<<<nc, 32, 0, st>>>((const XzbCrcJob *)(sm + off_crcjobs), sm + off_crcv, nullptr);
			CK(cudaMemcpyAsync(got.data(), sm + off_crcv, 32 * (size_t)nc, cudaMemcpyDeviceToHost, st));
		} else {
			const bool c64 = c == 4;
			xzb_k_crc<<<nc, 1024, 0, st>>>((const XzbCrcJob *)(sm + off_crcjobs), c64 ? ctx->d_crc64 : ctx->d_crc32w, c64 ? ~0ull : 0xFFFFFFFFull, (uint64_t *)(sm + off_crcv), 1, nullptr);
			CK(cudaMemcpyAsync(got.data(), sm + off_crcv, 8 * (size_t)nc, cudaMemcpyDeviceToHost, st));
		}
		ctx->stats.gpu_launches += 1;
		CK(cudaStreamSynchronize(st));
		for (uint32_t k = 0; k < nc; ++k) {
			if (c == 10) memcpy(shas->data() + 32 * (size_t)who[k], got.data() + 32 * (size_t)k, 32);
			else memcpy(&crcs[who[k]], got.data() + 8 * (size_t)k, 8);
		}
	}
	CK(cudaEventRecord(ctx->ev[2], st));
	CK(cudaStreamSynchronize(st));
	CK(cudaGetLastError());
	ctx->stats.ms_decode += ev_ms(ctx->ev[0], ctx->ev[1]);
	ctx->stats.ms_other += ev_ms(ctx->ev[1], ctx->ev[2]);
	ctx->stats.n_blocks += B;
	return XZB_OK;
}

extern "C" int xzb_decode_blocks_device(xzb_ctx *ctx, const void *d_in, const uint64_t *comp_off, const uint64_t *comp_size,
		const uint64_t *uncomp_size, const uint64_t *out_off, const uint32_t *dict_size, uint32_t nblocks, uint32_t check, void *d_out,
		uint32_t *ret, uint64_t *check_out)
{
	cudaSetDevice(ctx->device);
	memset(&ctx->stats, 0, sizeof(ctx->stats));
	cudaStream_t st = ctx->stream;
	CK(cudaEventRecord(ctx->ev[6], st));
	std::vector<XzbDecJob> jobs(nblocks);
	for (uint32_t b = 0; b < nblocks; ++b) {
		if (comp_size[b] > 0xFFFFFFF0ull || uncomp_size[b] > 0xFFFFFFF0ull) return set_err(ctx, XZB_OPTIONS_ERROR, "block too large");
		jobs[b].in = (const uint8_t *)d_in + comp_off[b]; jobs[b].in_size = (uint32_t)comp_size[b];
		jobs[b].out = (uint8_t *)d_out + out_off[b]; jobs[b].out_limit = (uint32_t)uncomp_size[b];
		jobs[b].dict_size = dict_size[b];
	}
	if (check == 10 && check_out != nullptr) return set_err(ctx, XZB_UNSUPPORTED_CHECK, "check_out carries CRC values only; verify SHA-256 Streams with xzb_stream_decode*");
	std::vector<XzbDecResult> results; std::vector<uint64_t> crcs;
	int r = decode_batch(ctx, jobs, std::vector<uint32_t>(nblocks, check), results, crcs);
	if (r != XZB_OK) return r;
	for (uint32_t b = 0; b < nblocks; ++b) {
		uint32_t code = results[b].ret;
		if (code == XZB_NEED_INPUT || code == XZB_NEED_OUTPUT) code = XZB_DATA_ERROR;  // sizes are exact here
		if (code == XZB_OK && (results[b].in_used != jobs[b].in_size || results[b].out_used != jobs[b].out_limit)) code = XZB_DATA_ERROR;
		ret[b] = code;
		if (check_out) check_out[b] = crcs[b];
		ctx->stats.n_positions += results[b].out_used;
	}
	CK(cudaEventRecord(ctx->ev[7], st));
	CK(cudaStreamSynchronize(st));
	ctx->stats.ms_total = ev_ms(ctx->ev[6], ctx->ev[7]);
	return XZB_OK;
}

// lzma_raw_decoder_memusage() of the reference for an LZMA2 Block (filter_decoder.c:208-214 ->
// lzma2_decoder.c:291-295 -> lzma_decoder.c:1215-1220 -> lz_decoder.c:329-333, + LZMA_MEMUSAGE_BASE): the
// dictionary plus 66200 bytes of coder structures on the reference's LP64 build.  Walks the sized
// Block Headers of the Stream at `in` in order (host only) and reports the first Block that needs more
// than `limit` (*exceeds = 1), else the last Block's figure -- what lzma_memusage() returns after
// stream_decoder.c:199-232 has looked at it.  Blocks that do not parse end the walk (the decoder
// reports them).
extern "C" int xzb_stream_memusage(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint64_t limit, uint64_t *memusage, uint32_t *exceeds)
{
	*memusage = 32768;  // LZMA_MEMUSAGE_BASE, common.h:68
	*exceeds = 0;
	if (in_size < 12) return XZB_OK;
	const uint32_t csize = xzb_check_field_size(in[7] & 0x0F);
	uint64_t ip = 12;
	while (ip < in_size && in[ip] != 0x00) {
		XzbBlockHeader hb;
		if (xzb_block_header_decode(ctx->h_tab.crc32, in + ip, in_size - ip, &hb) != XZB_OK) break;
		*memusage = (uint64_t)hb.dict_size + 66200;
		if (*memusage > limit) { *exceeds = 1; break; }
		if (hb.comp == UINT64_MAX) break;  // unsized Block: its end is only known by decoding it
		const uint64_t total = hb.hsize + ((hb.comp + 3) & ~3ull) + csize;
		if (in_size - ip < total) break;
		ip += total;
	}
	return XZB_OK;
}

extern "C" int xzb_stream_decode_flags(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size,
		uint64_t *in_used, uint32_t flags);
extern "C" int xzb_stream_decode_ex(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size, uint64_t *in_used)
{
	return xzb_stream_decode_flags(ctx, in, in_size, out, out_cap, out_size, in_used, 0);
}

// One Stream with lzma_stream_buffer_decode()'s result mapping (common/stream_buffer_decoder.c:44-88):
// truncated input is XZB_DATA_ERROR, a too small output buffer XZB_BUF_ERROR.
extern "C" int xzb_stream_buffer_decode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size,
		uint64_t *in_used, uint32_t flags)
{
	int r = xzb_stream_decode_flags(ctx, in, in_size, out, out_cap, out_size, in_used, flags);
	if (r == XZB_BUF_ERROR && ctx->dec_buf_reason == 1) r = XZB_DATA_ERROR;
	return r;
}

extern "C" int xzb_stream_decode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size)
{
	uint64_t used = 0;
	return xzb_stream_decode_ex(ctx, in, in_size, out, out_cap, out_size, &used);
}

extern "C" int xzb_stream_decode_prior(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size,
		uint64_t *in_used, uint32_t flags, const xzb_index_record *prior, uint64_t n_prior);
extern "C" int xzb_stream_decode_flags(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size,
		uint64_t *in_used, uint32_t flags)
{
	return xzb_stream_decode_prior(ctx, in, in_size, out, out_cap, out_size, in_used, flags, nullptr, 0);
}

// One Stream in flight in decode_streams(): the caller's view, and the decoder's cursor over it (xzb_dec_stream.cuh).
struct XzbDecStream {
	const uint8_t *in; uint64_t in_size;     // host
	uint8_t *out; uint64_t out_cap;          // host
	uint32_t flags;
	const xzb_index_record *prior; uint64_t n_prior;  // see xzb_stream_decode_prior
	XzbDecCursor c;
	std::vector<xzb_index_record> recs;
	std::vector<XzbDecBlk> blks;             // the Blocks of the current round
	uint64_t d_in = 0, d_out = 0;            // its input / output in ctx->dec_in / ctx->dec_out
	size_t job0 = 0;
};

// Decodes the Streams S side by side.  Their inputs go to HBM in one copy of the span they cover; each round scans the
// next run of sized Blocks of every unfinished Stream (an unsized Block gets a round of its own), decodes all of them
// with one decode_batch (at most 4096 Blocks per launch), and validates each Stream's Blocks in Stream order.  Returns
// XZB_OK or an error of the whole call (device); the Streams' own verdicts are in S.
static int decode_streams(xzb_ctx *ctx, std::vector<XzbDecStream> &S)
{
	cudaStream_t st = ctx->stream;
	const uint32_t *crc32 = ctx->h_tab.crc32;
	const uint8_t *lo = nullptr, *hi = nullptr;
	uint64_t out_total = 0;
	for (XzbDecStream &s : S) {
		xzb_dec_init(s.c, s.in_size, s.out_cap, s.flags, s.n_prior);
		s.recs.assign(s.prior, s.prior + s.n_prior);
		if (!xzb_dec_header(s.c, s.in, crc32)) continue;
		if (lo == nullptr || s.in < lo) lo = s.in;
		if (hi == nullptr || s.in + s.in_size > hi) hi = s.in + s.in_size;
		s.d_out = out_total;
		out_total += (s.out_cap + 64 + 255) & ~255ull;
	}
	if (lo == nullptr) return XZB_OK;
	CK(cudaEventRecord(ctx->ev[6], st));
	EN(ctx->dec_in, (size_t)(hi - lo) + 64);
	CK(cudaEventRecord(ctx->ev[8], st));
	CK(cudaMemcpyAsync(ctx->dec_in.p, lo, (size_t)(hi - lo), cudaMemcpyHostToDevice, st));
	CK(cudaEventRecord(ctx->ev[9], st));
	const uint8_t *d_in = (const uint8_t *)ctx->dec_in.p;
	EN(ctx->dec_out, out_total);
	uint8_t *d_out = (uint8_t *)ctx->dec_out.p;
	for (XzbDecStream &s : S) s.d_in = (uint64_t)(s.in - lo);

	for (;;) {
		std::vector<XzbDecJob> jobs;
		std::vector<uint32_t> checks;
		std::vector<XzbBlockHeader> hdrs;
		std::vector<XzbDecStream *> round;
		bool any_chain = false;
		for (XzbDecStream &s : S) {
			if (s.c.done || jobs.size() >= 4096) continue;
			// the run's length first, as xzb_k_dec_scan learns it, then the run into an array of that size
			XzbDecCursor probe = s.c;
			const uint32_t nb = xzb_dec_scan(probe, s.in, crc32, nullptr, (uint32_t)(4096 - jobs.size()), s.recs.data());
			if (nb == 0) { s.c = probe; continue; }
			s.blks.resize(nb);
			xzb_dec_scan(s.c, s.in, crc32, s.blks.data(), nb, s.recs.data());
			s.job0 = jobs.size();
			for (uint32_t b = 0; b < nb; ++b) {
				const XzbDecBlk &k = s.blks[b];
				XzbDecJob j;
				j.in = d_in + s.d_in + k.hdr_off + k.hb.hsize; j.in_size = k.in_avail;
				j.out = d_out + s.d_out + k.out_off; j.out_limit = k.out_limit; j.dict_size = k.hb.dict_size;
				jobs.push_back(j);
				checks.push_back(xzb_dec_check_computed(s.c));
				hdrs.push_back(k.hb);
				any_chain = any_chain || k.hb.n_pre != 0;
			}
			round.push_back(&s);
		}
		if (jobs.empty()) break;
		std::vector<XzbDecResult> results; std::vector<uint64_t> crcs; std::vector<uint8_t> shas;
		int r = decode_batch(ctx, jobs, checks, results, crcs, &shas, any_chain ? &hdrs : nullptr);
		if (r != XZB_OK) return r;
		for (XzbDecStream *sp : round) {
			XzbDecStream &s = *sp;
			const bool sha = s.c.check == 10;
			const uint8_t *chk = sha ? shas.data() + 32 * s.job0 : (const uint8_t *)(crcs.data() + s.job0);
			s.recs.resize(s.c.n_recs + s.c.nb);  // a round appends at most one record per Block
			ctx->stats.n_positions += xzb_dec_settle(s.c, s.in, crc32, s.blks.data(), results.data() + s.job0, chk, sha ? 32 : 8,
					s.recs.data(), s.recs.size());
		}
	}
	// bytes of successfully validated blocks are delivered even when a later block fails
	CK(cudaEventRecord(ctx->ev[10], st));
	for (const XzbDecStream &s : S)
		if (s.c.out_size > 0) CK(cudaMemcpyAsync(s.out, d_out + s.d_out, s.c.out_size, cudaMemcpyDeviceToHost, st));
	CK(cudaEventRecord(ctx->ev[11], st));
	CK(cudaEventRecord(ctx->ev[7], st));
	CK(cudaStreamSynchronize(st));
	ctx->stats.ms_h2d = ev_ms(ctx->ev[8], ctx->ev[9]);
	ctx->stats.ms_d2h = ev_ms(ctx->ev[10], ctx->ev[11]);
	ctx->stats.ms_total = ev_ms(ctx->ev[6], ctx->ev[7]);
	return XZB_OK;
}

// The same with the Index records of Blocks that were already decoded (and removed from `in`) by earlier
// calls: a caller that streams a long Stream hands its complete Blocks over in parts and gives the last
// part -- whatever Blocks remain, the real Index and the Stream Footer -- together with the records of
// all earlier parts, so that the Index is verified against every Block of the Stream.
extern "C" int xzb_stream_decode_prior(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint8_t *out, uint64_t out_cap, uint64_t *out_size,
		uint64_t *in_used, uint32_t flags, const xzb_index_record *prior, uint64_t n_prior)
{
	*in_used = 0;
	*out_size = 0;
	cudaSetDevice(ctx->device);
	memset(&ctx->stats, 0, sizeof(ctx->stats));
	ctx->err[0] = 0;
	// XZB_BUF_ERROR has two causes that the one-shot API tells apart (stream_buffer_decoder.c:56-71):
	// 1 = the input ended early, 2 = the output buffer is too small.
	ctx->dec_buf_reason = 1;
	std::vector<XzbDecStream> S(1);
	S[0].in = in; S[0].in_size = in_size; S[0].out = out; S[0].out_cap = out_cap; S[0].flags = flags;
	S[0].prior = prior; S[0].n_prior = n_prior;
	const int r = decode_streams(ctx, S);
	if (r != XZB_OK) return r;
	*in_used = S[0].c.in_used;
	*out_size = S[0].c.out_size;
	ctx->dec_buf_reason = S[0].c.buf_reason;
	return S[0].c.ret;
}

// n independent Streams with xzb_stream_buffer_decode()'s result mapping per item.  Items go to the device in groups
// whose inputs and output slots fit the memory budget.
extern "C" int xzb_stream_buffer_decode_batch(xzb_ctx *ctx, uint32_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_size,
		uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint64_t *in_used, uint32_t *ret, uint32_t flags)
{
	cudaSetDevice(ctx->device);
	memset(&ctx->stats, 0, sizeof(ctx->stats));
	ctx->err[0] = 0;
	size_t free_b = 0, total_b = 0;
	cudaMemGetInfo(&free_b, &total_b);
	const uint64_t budget = (uint64_t)((free_b + ctx->dec_in.cap + ctx->dec_out.cap) * 0.85);
	xzb_stats sum;
	memset(&sum, 0, sizeof(sum));
	for (uint32_t i0 = 0; i0 < n;) {
		std::vector<XzbDecStream> S;
		uint64_t lo = UINT64_MAX, hi = 0, outs = 0;
		uint32_t i = i0;
		for (; i < n; ++i) {
			const uint64_t l = std::min(lo, in_off[i]), h = std::max(hi, in_off[i] + in_size[i]), o = outs + ((out_cap[i] + 64 + 255) & ~255ull);
			if (i > i0 && (h - l) + o > budget) break;
			lo = l; hi = h; outs = o;
			XzbDecStream s;
			s.in = in + in_off[i]; s.in_size = in_size[i]; s.out = out + out_off[i]; s.out_cap = out_cap[i]; s.flags = flags;
			s.prior = nullptr; s.n_prior = 0;
			S.push_back(std::move(s));
		}
		const int r = decode_streams(ctx, S);
		if (r != XZB_OK) return r;
		for (uint32_t k = 0; k < S.size(); ++k) {
			int code = S[k].c.ret;
			if (code == XZB_BUF_ERROR && S[k].c.buf_reason == 1) code = XZB_DATA_ERROR;   // as xzb_stream_buffer_decode()
			ret[i0 + k] = (uint32_t)code; out_size[i0 + k] = S[k].c.out_size; in_used[i0 + k] = S[k].c.in_used;
		}
		sum.ms_total += ctx->stats.ms_total; sum.ms_h2d += ctx->stats.ms_h2d; sum.ms_d2h += ctx->stats.ms_d2h;
		sum.ms_decode += ctx->stats.ms_decode; sum.ms_other += ctx->stats.ms_other; sum.gpu_launches += ctx->stats.gpu_launches;
		sum.n_blocks += ctx->stats.n_blocks; sum.n_positions += ctx->stats.n_positions;
		memset(&ctx->stats, 0, sizeof(ctx->stats));
		i0 = i;
	}
	ctx->stats = sum;
	return XZB_OK;
}

// ------------------------------------------------------------------------------------
// Decode, device-resident batch
// ------------------------------------------------------------------------------------
static const uint32_t XZB_DEC_ROUND_JOBS = 65536;  // Blocks decoded per round at most (the job area's capacity)

static size_t dec_align(size_t v) { return (v + 255) & ~(size_t)255; }

// HBM of one round's job area of `cap` jobs.
static size_t dec_job_area(uint32_t cap)
{
	return dec_align(sizeof(XzbDecCounters)) + dec_align(sizeof(XzbDecBlk) * cap) + dec_align(sizeof(XzbDecJob) * cap)
		+ dec_align(sizeof(XzbDecResult) * cap) + dec_align(sizeof(XzbFiltJob) * 3 * (size_t)cap) + dec_align(sizeof(XzbCrcJob) * 3 * (size_t)cap)
		+ dec_align(8 * 2 * (size_t)cap) + dec_align(32 * (size_t)cap);
}
static const uint64_t XZB_DEC_ITEM_BYTES = sizeof(XzbDecCursor) + sizeof(XzbDecItem) + sizeof(XzbDecRound) + sizeof(XzbDecOut);

// One group of items, all rounds.  Fills out_size / in_used / ret of items [i0, i0 + ng).
static int decode_group_device(xzb_ctx *ctx, uint32_t ng, const uint8_t *d_in, const uint64_t *in_off, const uint64_t *in_size,
		uint8_t *d_out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint64_t *in_used, uint32_t *ret, uint32_t flags)
{
	cudaStream_t st = ctx->stream;
	uint64_t recs_total = 0;
	for (uint32_t i = 0; i < ng; ++i) recs_total += xzb_dec_rec_bound(in_size[i]);
	const uint32_t cap = (uint32_t)std::min<uint64_t>(XZB_DEC_ROUND_JOBS, recs_total);
	// layout: counters, job area, then the per-item arrays and record areas
	size_t o = 0;
	auto take = [&](size_t bytes) { const size_t at = o; o += dec_align(bytes); return at; };
	const size_t o_cnt = take(sizeof(XzbDecCounters)), o_blk = take(sizeof(XzbDecBlk) * cap), o_job = take(sizeof(XzbDecJob) * cap);
	const size_t o_res = take(sizeof(XzbDecResult) * cap), o_filt = take(sizeof(XzbFiltJob) * 3 * (size_t)cap);
	const size_t o_cj = take(sizeof(XzbCrcJob) * 3 * (size_t)cap), o_crcv = take(8 * 2 * (size_t)cap), o_shav = take(32 * (size_t)cap);
	const size_t o_cur = take(sizeof(XzbDecCursor) * ng), o_item = take(sizeof(XzbDecItem) * ng), o_round = take(sizeof(XzbDecRound) * ng);
	const size_t o_out = take(sizeof(XzbDecOut) * ng), o_recs = take(sizeof(xzb_index_record) * recs_total);
	EN(ctx->decs, o);
	uint8_t *base = (uint8_t *)ctx->decs.p;
	XzbDecCounters *cnt = (XzbDecCounters *)(base + o_cnt);
	XzbDecBlk *blks = (XzbDecBlk *)(base + o_blk);
	XzbDecJob *jobs = (XzbDecJob *)(base + o_job);
	XzbDecResult *res = (XzbDecResult *)(base + o_res);
	XzbFiltJob *filt = (XzbFiltJob *)(base + o_filt);
	XzbCrcJob *cj = (XzbCrcJob *)(base + o_cj);
	uint64_t *crcv = (uint64_t *)(base + o_crcv);
	uint8_t *shav = base + o_shav;
	XzbDecCursor *cur = (XzbDecCursor *)(base + o_cur);
	XzbDecItem *items = (XzbDecItem *)(base + o_item);
	XzbDecRound *round = (XzbDecRound *)(base + o_round);
	XzbDecOut *outs = (XzbDecOut *)(base + o_out);
	xzb_index_record *recs = (xzb_index_record *)(base + o_recs);
	// the cursors and where each item's bytes are: per-item metadata, no item data
	std::vector<XzbDecCursor> hc(ng);
	std::vector<XzbDecItem> hi(ng);
	uint64_t r0 = 0;
	for (uint32_t i = 0; i < ng; ++i) {
		xzb_dec_init(hc[i], in_size[i], out_cap[i], flags, 0);
		const uint64_t rc = xzb_dec_rec_bound(in_size[i]);
		hi[i] = XzbDecItem{ d_in + in_off[i], d_out + out_off[i], recs + r0, rc };
		r0 += rc;
	}
	CK(cudaMemcpyAsync(cur, hc.data(), sizeof(XzbDecCursor) * ng, cudaMemcpyHostToDevice, st));
	CK(cudaMemcpyAsync(items, hi.data(), sizeof(XzbDecItem) * ng, cudaMemcpyHostToDevice, st));
	CK(cudaMemsetAsync(cnt, 0, sizeof(XzbDecCounters), st));
	const uint32_t grid_items = (ng + 127) / 128;
	XzbDecCounters h;
	for (;;) {
		CK(cudaMemsetAsync(cnt, 0, offsetof(XzbDecCounters, positions), st));
		xzb_k_dec_scan<<<grid_items, 128, 0, st>>>(cur, items, ng, ctx->d_crc32, cap, blks, jobs, round, cnt);
		CK(cudaMemcpyAsync(&h, cnt, sizeof(h), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		ctx->stats.gpu_launches += 1;
		const uint32_t nj = std::min(h.njobs, cap);
		if (nj == 0) break;   // every item finished at its header or its Index
		CK(cudaEventRecord(ctx->ev[0], st));
		xzb_k_decode<<<nj, 32, sizeof(XzbDec), st>>>(jobs, res);
		CK(cudaEventRecord(ctx->ev[1], st));
		xzb_k_dec_prep<<<grid_items, 128, 0, st>>>(cur, round, ng, blks, jobs, res, cap, filt, cj, cnt);
		ctx->stats.gpu_launches += 2;
		// Delta / BCJ behind LZMA2 (common/filter_decoder.c:44-139), undone in reverse chain order before the checks
		for (uint32_t lvl = 0; lvl < h.depth; ++lvl) { xzb_k_filter<<<nj, 256, 0, st>>>(filt + (size_t)lvl * cap, 0); ctx->stats.gpu_launches += 1; }
		for (uint32_t list = 0; list < 3; ++list) {
			if (!(h.checks & (1u << list))) continue;
			if (list == 2) xzb_k_sha256<<<nj, 32, 0, st>>>(cj + 2 * (size_t)cap, shav, &cnt->nchk[2]);
			else xzb_k_crc<<<nj, 1024, 0, st>>>(cj + (size_t)list * cap, list ? ctx->d_crc64 : ctx->d_crc32w, list ? ~0ull : 0xFFFFFFFFull,
					crcv + (size_t)list * cap, 1, &cnt->nchk[list]);
			ctx->stats.gpu_launches += 1;
		}
		xzb_k_dec_settle<<<grid_items, 128, 0, st>>>(cur, items, round, ng, ctx->d_crc32, blks, res, cap, crcv, shav, cnt);
		CK(cudaEventRecord(ctx->ev[2], st));
		CK(cudaMemcpyAsync(&h, cnt, sizeof(h), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		CK(cudaGetLastError());
		ctx->stats.gpu_launches += 1;
		ctx->stats.ms_decode += ev_ms(ctx->ev[0], ctx->ev[1]);
		ctx->stats.n_blocks += nj;
		if (h.live == 0) break;
	}
	xzb_k_dec_results<<<grid_items, 128, 0, st>>>(cur, ng, outs);
	ctx->stats.gpu_launches += 1;
	std::vector<XzbDecOut> ho(ng);
	CK(cudaMemcpyAsync(ho.data(), outs, sizeof(XzbDecOut) * ng, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(&h, cnt, sizeof(h), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	CK(cudaGetLastError());
	ctx->stats.n_positions += h.positions;
	for (uint32_t i = 0; i < ng; ++i) { ret[i] = ho[i].ret; out_size[i] = ho[i].out_size; in_used[i] = ho[i].in_used; }
	return XZB_OK;
}

// xzb_stream_buffer_decode_batch with the Streams and the output slots in device memory: the container is read on the
// GPU (xzb_dec_stream.cuh) and every Block decodes straight into its item's slot.  Items go in groups whose cursors
// and Index record areas fit the memory budget beside one round's job area.
extern "C" int xzb_stream_buffer_decode_batch_device(xzb_ctx *ctx, uint32_t n, const uint8_t *d_in, const uint64_t *in_off,
		const uint64_t *in_size, uint8_t *d_out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint64_t *in_used,
		uint32_t *ret, uint32_t flags)
{
	cudaSetDevice(ctx->device);
	memset(&ctx->stats, 0, sizeof(ctx->stats));
	ctx->err[0] = 0;
	if (n == 0) return XZB_OK;
	cudaStream_t st = ctx->stream;
	CK(cudaEventRecord(ctx->ev[6], st));
	size_t free_b = 0, total_b = 0;
	cudaMemGetInfo(&free_b, &total_b);
	const uint64_t avail = (uint64_t)((free_b + ctx->decs.cap) * 0.85), jobs = dec_job_area(XZB_DEC_ROUND_JOBS);
	std::vector<uint32_t> start;
	xzb_plan_dec_groups(in_size, n, XZB_DEC_ITEM_BYTES, avail > jobs ? avail - jobs : 0, &start);
	for (size_t g = 0; g + 1 < start.size(); ++g) {
		const uint32_t i0 = start[g], ng = start[g + 1] - i0;
		const int r = decode_group_device(ctx, ng, d_in, in_off + i0, in_size + i0, d_out, out_off + i0, out_cap + i0, out_size + i0,
				in_used + i0, ret + i0, flags);
		if (r != XZB_OK) return r;
	}
	CK(cudaEventRecord(ctx->ev[7], st));
	CK(cudaStreamSynchronize(st));
	ctx->stats.ms_total = ev_ms(ctx->ev[6], ctx->ev[7]);
	ctx->stats.ms_other = std::max(0.0, ctx->stats.ms_total - ctx->stats.ms_decode);
	return XZB_OK;
}

static_assert(sizeof(FS<false>) <= XZB_SOLO_SMEM && 2 * XZB_SOLO_SMEM > 228 * 1024 && XZB_SOLO_SMEM <= 227 * 1024,
		"the two-warp fast-mode kernel must hold its state and take more than half of an SM's 228 KB of shared memory");
static_assert(sizeof(DS) <= 227 * 1024, "parser shared memory exceeds the 227 KB per-CTA limit of sm_90");
