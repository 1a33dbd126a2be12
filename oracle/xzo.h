/*
 * oracle/xzo.h -- CPU oracle for the LZMA2 / .xz block path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is a plain-C restatement of the reference's
 * algorithm (tukaani-project/xz @ 28a66a3d, liblzma 5.8.3) used by tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline leg as the *checker*.
 * Nothing under xz_b200/ (the product) may include, link or call it.
 *
 * Parity of this restatement is PINNED: tests/test_oracle_vs_ref.py compares it
 * byte-for-byte with the unmodified reference (oracle/_ref/liblzma_ref.so, built by
 * oracle/Makefile.ref from /root/reference) and with the reference's own golden
 * vectors (tests/golden/).
 */
#ifndef XZO_H
#define XZO_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* LZMA_MF_* / LZMA_MODE_* values, src/liblzma/api/lzma/lzma12.h:58-138 */
enum { XZO_MF_HC3 = 0x03, XZO_MF_HC4 = 0x04, XZO_MF_BT2 = 0x12, XZO_MF_BT3 = 0x13, XZO_MF_BT4 = 0x14 };
enum { XZO_MODE_FAST = 1, XZO_MODE_NORMAL = 2 };
/* lzma_check, src/liblzma/api/lzma/check.h:27-66 */
enum { XZO_CHECK_NONE = 0, XZO_CHECK_CRC32 = 1, XZO_CHECK_CRC64 = 4 };
#define XZO_PRESET_EXTREME 0x80000000u

/* lzma_ret subset, src/liblzma/api/lzma/base.h:55-271 */
enum {
	XZO_OK = 0, XZO_STREAM_END = 1, XZO_UNSUPPORTED_CHECK = 3, XZO_MEM_ERROR = 5,
	XZO_FORMAT_ERROR = 7, XZO_OPTIONS_ERROR = 8, XZO_DATA_ERROR = 9,
	XZO_BUF_ERROR = 10, XZO_PROG_ERROR = 11,
};

/* The subset of lzma_options_lzma (lzma12.h:216-525) the path uses. */
typedef struct {
	uint32_t dict_size;
	uint32_t lc, lp, pb;
	uint32_t mode;      /* XZO_MODE_* */
	uint32_t nice_len;
	uint32_t mf;        /* XZO_MF_* */
	uint32_t depth;     /* 0 = default */
} xzo_lzma_options;

/* lzma_lzma_preset(), src/liblzma/lzma/lzma_encoder_presets.c:16-63. Returns 1 on error. */
int xzo_lzma_preset(xzo_lzma_options *opt, uint32_t preset);

/* Counters the roofline arithmetic needs (SURVEY.md section 8d). */
typedef struct {
	uint64_t n_pos;        /* positions run through the match finder */
	uint64_t n_nodes;      /* hash-chain / binary-tree nodes visited */
	uint64_t n_cmp_bytes;  /* bytes compared inside memcmplen calls of the match finder */
	uint64_t n_pairs;      /* (len,dist) pairs reported */
	uint64_t n_symbols;    /* LZMA symbols emitted */
	uint64_t n_chunks_lzma, n_chunks_raw;
	uint64_t n_raw_with_read_ahead; /* D12 probe: raw chunk taken with read_ahead != 0 */
	uint64_t n_raw_ahead_then_lzma; /* of those, the ones the next chunk of the same Block codes as LZMA */
} xzo_counters;

/* lzma_block_buffer_bound64(), src/liblzma/common/block_buffer_encoder.c:56-71 */
uint64_t xzo_block_bound(uint64_t uncompressed_size);

/*
 * One .xz Block exactly as worker_encode() produces it
 * (src/liblzma/common/stream_encoder_mt.c:218-359): Block Header (sizes present),
 * LZMA2 data, Block Padding, Check.  block_size is lzma_mt.block_size (fixes the
 * header size and the out buffer bound).  out must hold xzo_block_bound(block_size).
 * Returns XZO_OK and sets out_size / unpadded / uncompressed.
 */
int xzo_block_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint32_t check, uint64_t block_size, uint8_t *out, size_t *out_size,
		uint64_t *unpadded_size, xzo_counters *ctr);

/* Whole .xz Stream as lzma_stream_encoder_mt + lzma_code(FINISH) produce it
 * (stream_encoder_mt.c:716-888).  Returns XZO_OK or an error. */
int xzo_stream_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint32_t check, uint64_t block_size, uint8_t *out, size_t out_cap,
		size_t *out_size, xzo_counters *ctr);
size_t xzo_stream_bound(size_t in_size, uint64_t block_size);

/* One-shot buffer API: lzma_stream_buffer_encode / lzma_easy_buffer_encode (common/stream_buffer_encoder.c:43-140):
 * one Block over the whole input, lzma_block_buffer_encode framing. */
size_t xzo_stream_buffer_bound(size_t uncompressed_size);
int xzo_stream_buffer_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt, uint32_t check,
		uint8_t *out, size_t out_cap, size_t *out_size);

/* Stream framing pieces (stream_flags_encoder.c:29-85, index_encoder.c:43-165). */
size_t xzo_stream_header(uint8_t out[12], uint32_t check);
size_t xzo_stream_footer(uint8_t out[12], uint32_t check, uint64_t index_size);
size_t xzo_index_encode(const uint64_t *unpadded, const uint64_t *uncompressed,
		size_t count, uint8_t *out); /* out may be NULL to get the size */

/*
 * Match-finder dump: run mf_find at EVERY position of in[0..n) with the options'
 * match finder (lz_encoder_mf.c:21-79 semantics incl. the nice_len extension) and
 * return, for position p, counts[p], longest[p] and the pairs at
 * pairs[offsets[p] .. offsets[p]+counts[p]) as (len,dist) u32 pairs.
 * pairs_cap is in pairs; returns total number of pairs, or (uint64_t)-1 if cap exceeded.
 */
uint64_t xzo_mf_dump(const uint8_t *in, uint32_t n, const xzo_lzma_options *opt,
		uint32_t *counts, uint32_t *longest, uint64_t *offsets,
		uint32_t *pairs, uint64_t pairs_cap, xzo_counters *ctr);

/* MicroLZMA framing of the LZMA core, for the reference's encoder KAT (tests/test_microlzma.c:20-32). */
int xzo_microlzma_encode(const uint8_t *in, size_t in_size, const xzo_lzma_options *opt,
		uint8_t *out, size_t out_cap, size_t *out_size);

/* Optional symbol trace for diffing parses: (position, back, len) triples. */
void xzo_set_trace(uint32_t *triples, size_t cap_triples, size_t *count);

/* ---- decoder ---- */

/* Raw LZMA2 decode of one Block's compressed data (lzma2_decoder.c:55-230 +
 * lzma_decoder.c:234-1021): out_size must be the exact uncompressed size when
 * known, otherwise a capacity (exact=0).  Returns XZO_OK or XZO_DATA_ERROR. */
int xzo_lzma2_decode(const uint8_t *in, size_t in_size, uint32_t dict_size,
		uint8_t *out, size_t out_cap, size_t *out_size, size_t *in_used);

/* Whole-stream decode (stream_decoder.c:101-378, block_decoder.c:64-200,
 * index_hash.c) with flags = 0: decodes the first Stream and stops there, as
 * lzma_stream_decoder(strm, UINT64_MAX, 0) + lzma_code(LZMA_FINISH) does.  Only the
 * LZMA2-only filter chain and CRC32/CRC64/None checks are in scope (others:
 * XZO_OPTIONS_ERROR / XZO_UNSUPPORTED_CHECK). */
int xzo_stream_decode(const uint8_t *in, size_t in_size, uint8_t *out, size_t out_cap,
		size_t *out_size);

/* Checks (check/crc32_fast.c, crc64_fast.c; KATs tests/test_check.c:74,112). */
uint32_t xzo_crc32(const uint8_t *buf, size_t size, uint32_t crc);
uint64_t xzo_crc64(const uint8_t *buf, size_t size, uint64_t crc);
void xzo_sha256(const uint8_t *buf, size_t size, uint8_t out[32]); /* FIPS 180-4; reference: check/sha256.c */


#ifdef __cplusplus
}
#endif
#endif
