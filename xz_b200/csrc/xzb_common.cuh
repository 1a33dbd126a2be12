// xzb_common.cuh -- shared definitions for the H100 LZMA2 block path.
//
// Product code (sm_90a).  Functions marked XZB_HD also compile for the host so that
// tests/hostsim can single-step the very same logic on a CPU box without a GPU; the host
// build is a debugging harness under tests/, never a fallback of the product.
#pragma once

#include <stdint.h>
#include <stddef.h>

#ifdef __CUDACC__
#define XZB_HD __host__ __device__ __forceinline__
#define XZB_HD_NOINLINE __host__ __device__ __noinline__
#define XZB_HDM __host__ __device__ __forceinline__
#else
#define XZB_HD static inline
#define XZB_HD_NOINLINE static
#define XZB_HDM inline
#endif

// ---- constants of the LZMA model (reference: lzma/lzma_common.h:55-240,
//      lzma/lzma_encoder_private.h:29-36, lzma/lzma2_encoder.h:19-29) ----
#define XZB_REPS 4
#define XZB_MATCH_LEN_MIN 2
#define XZB_MATCH_LEN_MAX 273
#define XZB_OPTS 4096
#define XZB_STATES 12
#define XZB_LIT_STATES 7
#define XZB_POS_STATES_MAX 16
#define XZB_LEN_LOW 8
#define XZB_LEN_MID 8
#define XZB_LEN_HIGH 256
#define XZB_LEN_SYMBOLS (XZB_LEN_LOW + XZB_LEN_MID + XZB_LEN_HIGH)
#define XZB_DIST_STATES 4
#define XZB_DIST_SLOTS 64
#define XZB_DIST_MODEL_START 4
#define XZB_DIST_MODEL_END 14
#define XZB_FULL_DISTANCES 128
#define XZB_ALIGN_BITS 4
#define XZB_ALIGN_SIZE 16
#define XZB_ALIGN_MASK 15
#define XZB_INFINITY_PRICE (1u << 30)
#define XZB_LZMA2_CHUNK_MAX (1u << 16)
#define XZB_LZMA2_UNCOMPRESSED_MAX (1u << 21)
#define XZB_LZMA2_HEADER_MAX 6
#define XZB_LOOP_INPUT_MAX (XZB_OPTS + 1)
#define XZB_BACK_LITERAL 0xFFFFFFFFu

#define XZB_H2_SIZE 1024u
#define XZB_H3_SIZE 65536u
#define XZB_NONE 0xFFFFFFFFu

// lzma_match_finder / lzma_mode values (api/lzma/lzma12.h:58-138)
#define XZB_MF_HC3 0x03
#define XZB_MF_HC4 0x04
#define XZB_MF_BT2 0x12
#define XZB_MF_BT3 0x13
#define XZB_MF_BT4 0x14
#define XZB_MODE_FAST 1
#define XZB_MODE_NORMAL 2

// lzma_ret values we produce (api/lzma/base.h:55-271)
#define XZB_OK 0
#define XZB_STREAM_END 1
#define XZB_UNSUPPORTED_CHECK 3
#define XZB_MEM_ERROR 5
#define XZB_FORMAT_ERROR 7
#define XZB_OPTIONS_ERROR 8
#define XZB_DATA_ERROR 9
#define XZB_BUF_ERROR 10
#define XZB_PROG_ERROR 11
#define XZB_MF_STALL 102            // internal: parser watchdog, see WarpEncT::mf_wait
#define XZB_MF_STALL_NS 30000000000ull  // no match-finder progress for this long = kernels are not running side by side

typedef uint16_t xzb_prob;

// Derived match-finder / coder constants for one filter configuration
// (lz/lz_encoder.c:191-368 lz_encoder_prepare, lzma/lzma_encoder.c:486-502, 601-707).
struct XzbParams {
	uint32_t dict_size, lc, lp, pb, mode, nice_len, mf, depth;  // as given (depth resolved)
	uint32_t hash_bytes, is_bt, cyclic_size, hash_mask;
	uint32_t dist_table_size;  // normal mode
	uint32_t len_table_size;   // nice_len + 1 - MATCH_LEN_MIN (normal mode)
	uint32_t mstride;          // pairs stored inline per position in the match store
	uint8_t dict_prop;         // LZMA2 dictionary size property byte
	uint8_t lclppb;            // (pb*5+lp)*9+lc
	// filters in front of LZMA2 (Delta / BCJ): their Filter Flags as they go into every Block Header
	uint8_t n_pre, ff_len;
	uint8_t ff[18];
};

// Read-only tables in device memory (crc32 table doubles as the match-finder hash table,
// lz/lz_encoder_hash.h:30-39; price table rangecoder/price_tablegen.c:28-56).
struct XzbTables {
	const uint32_t *crc32;   // [256]
	const uint64_t *crc64;   // [256]
	const uint8_t *prices;   // [128]
};

// get_dist_slot / get_dist_slot_2, lzma/fastpos.h:77-136 (bsr form)
XZB_HD uint32_t xzb_clz32(uint32_t v)
{
#ifdef __CUDA_ARCH__
	return (uint32_t)__clz((int)v);
#else
	return (uint32_t)__builtin_clz(v);
#endif
}
XZB_HD uint32_t xzb_dist_slot(uint32_t dist)
{
	if (dist <= 4) return dist;
	const uint32_t i = 31 - xzb_clz32(dist);
	return (i + i) + ((dist >> (i - 1)) & 1);
}

// get_dist_state, lzma_common.h:133-136
XZB_HD uint32_t xzb_dist_state(uint32_t len) { return len < XZB_DIST_STATES + XZB_MATCH_LEN_MIN ? len - XZB_MATCH_LEN_MIN : XZB_DIST_STATES - 1; }

XZB_HD uint32_t xzb_min(uint32_t a, uint32_t b) { return a < b ? a : b; }
XZB_HD uint32_t xzb_max(uint32_t a, uint32_t b) { return a > b ? a : b; }

// common/memcmplen.h:52-190: first index >= len at which a and b differ, capped at limit.
XZB_HD uint32_t xzb_memcmplen(const uint8_t *a, const uint8_t *b, uint32_t len, uint32_t limit)
{
	while (len < limit && a[len] == b[len]) ++len;
	return len;
}


// 4 bytes at an arbitrary address from two aligned word loads (reads up to 7 bytes past p).
XZB_HD uint32_t xzb_ld32u(const uint8_t *p)
{
#ifdef __CUDA_ARCH__
	const uintptr_t a = (uintptr_t)p;
	const uint32_t *w = (const uint32_t *)(a & ~(uintptr_t)3);
	return __funnelshift_r(w[0], w[1], (uint32_t)(a & 3) * 8);
#else
	return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
#endif
}
XZB_HD uint32_t xzb_ctz32(uint32_t v)
{
#ifdef __CUDA_ARCH__
	return (uint32_t)__ffs((int)v) - 1;
#else
	return (uint32_t)__builtin_ctz(v);
#endif
}

// Same result as xzb_memcmplen, 4 bytes per step (the memcmplen.h:82-106 idea on 32-bit words).
// `room` = bytes that may be read starting at a (a is the later of the two pointers): the word
// path is only used while its 8-byte read window stays inside it.
XZB_HD uint32_t xzb_memcmplen_w(const uint8_t *a, const uint8_t *b, uint32_t len, uint32_t limit, uint32_t room)
{
	while (len + 4 <= limit && len + 8 <= room) {
		const uint32_t x = xzb_ld32u(a + len) ^ xzb_ld32u(b + len);
		if (x != 0) return len + (xzb_ctz32(x) >> 3);
		len += 4;
	}
	while (len < limit && a[len] == b[len]) ++len;
	return len;
}

// Like xzb_memcmplen_w, and when the result is < limit also hands back the two differing bytes
// (a[result], b[result]) taken from the words it already loaded, so the caller's follow-up
// "which side is smaller" test (bt_find_func, lz_encoder_mf.c:500) costs no further memory access.
XZB_HD uint32_t xzb_memcmplen_w2(const uint8_t *a, const uint8_t *b, uint32_t len, uint32_t limit, uint32_t room, uint32_t *ba, uint32_t *bb)
{
	while (len + 4 <= limit && len + 8 <= room) {
		const uint32_t wa = xzb_ld32u(a + len), wb = xzb_ld32u(b + len);
		const uint32_t x = wa ^ wb;
		if (x != 0) {
			const uint32_t k = xzb_ctz32(x) >> 3;
			*ba = (wa >> (8 * k)) & 0xFF; *bb = (wb >> (8 * k)) & 0xFF;
			return len + k;
		}
		len += 4;
	}
	while (len < limit) {
		const uint32_t ca = a[len], cb = b[len];
		if (ca != cb) { *ba = ca; *bb = cb; return len; }
		++len;
	}
	return len;
}
