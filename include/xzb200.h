/*
 * xzb200.h -- C ABI of the H100-native LZMA2 / .xz block path (libxzb200.so).
 *
 * Plain C, plain pointers and sizes; no CUDA or torch types.  Each entry point names the
 * reference interface it stands in for (paths relative to the reference's src/liblzma/).
 * The natural cut is whole-Block: a batch of independent .xz Blocks goes in, finished
 * Blocks plus their Index records come out -- exactly what one worker thread of the
 * reference's threaded coders does per Block.
 *
 * All functions return an lzma_ret-compatible code (api/lzma/base.h:55-271):
 *   0 LZMA_OK, 3 LZMA_UNSUPPORTED_CHECK, 5 LZMA_MEM_ERROR, 7 LZMA_FORMAT_ERROR,
 *   8 LZMA_OPTIONS_ERROR, 9 LZMA_DATA_ERROR, 10 LZMA_BUF_ERROR, 11 LZMA_PROG_ERROR.
 * There is no CPU fallback: without a usable CUDA device xzb_ctx_create() fails with
 * LZMA_PROG_ERROR and nothing else can be called.
 */
#ifndef XZB200_H
#define XZB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct xzb_ctx xzb_ctx;

/* Subset of lzma_options_lzma that the LZMA2 encoder reads (api/lzma/lzma12.h:216-525). */
typedef struct {
	uint32_t dict_size, lc, lp, pb;
	uint32_t mode;     /* lzma_mode: 1 fast, 2 normal */
	uint32_t nice_len;
	uint32_t mf;       /* lzma_match_finder: 0x03 hc3, 0x04 hc4, 0x12 bt2, 0x13 bt3, 0x14 bt4 */
	uint32_t depth;
} xzb_lzma_options;

/* One Index record per Block (common/index.c:722 lzma_index_append arguments); this is the
 * 16-byte unit that ranks exchange with one NCCL all-gather to reassemble the Index. */
typedef struct {
	uint64_t unpadded_size;
	uint64_t uncompressed_size;
} xzb_index_record;

/* Timing and work counters of the last encode/decode call (device times from CUDA events on
 * the context's stream).  Used by bench.py for the roofline line. */
typedef struct {
	double ms_total;        /* whole call, device side */
	double ms_h2d, ms_d2h;  /* host<->device copies (host-buffer entry points only) */
	double ms_mf_prep;      /* hash keys + radix sorts + previous-occurrence scatter */
	double ms_mf;           /* match-finder kernel (xzb_k_hc / xzb_k_bt) */
	double ms_parse;        /* parser + range coder kernel */
	double ms_other;        /* crc, finalize, pack */
	double ms_decode;       /* decode kernel */
	uint64_t gpu_launches;  /* kernels launched by this library in the call */
	uint64_t n_blocks, n_positions, n_symbols, n_chunks_lzma, n_chunks_raw, n_fallback_blocks;
	uint64_t mf_bytes_algorithmic; /* SURVEY 8(d) B_mf lower bound: N_pos * (29|33) */
} xzb_stats;

/* lzma_lzma_preset(), lzma/lzma_encoder_presets.c:16-63.  Returns nonzero on bad preset. */
int xzb_lzma_preset(xzb_lzma_options *opt, uint32_t preset);

/* lzma_block_buffer_bound64(), common/block_buffer_encoder.c:56-71, and the size of the
 * largest .xz Stream xzb_stream_encode() can produce for in_size bytes. */
uint64_t xzb_block_bound(uint64_t uncompressed_size);
uint64_t xzb_stream_bound(uint64_t in_size, uint64_t block_size);

/* Create/destroy a context bound to CUDA device `device` (one per process/rank).
 * Stands in for the worker pool of stream_encoder_mt.c:362-595 / stream_decoder_mt.c. */
int xzb_ctx_create(xzb_ctx **ctx, int device);
void xzb_ctx_destroy(xzb_ctx *ctx);
/* CUDA devices visible to this process (0 when there is none). */
int xzb_device_count(void);

/* The filter-chain table of the path (common/filter_encoder.c:59-182, filter_decoder.c:44-139): LZMA2 is always the
 * last filter; up to three of these may stand in front of it.  Decoding needs no call: the chain is read from each
 * Block Header.  For encoding, xzb_ctx_set_filters() names the filters in front of LZMA2 for the following
 * xzb_encode_blocks_* calls (n = 0 switches back to LZMA2 alone). */
#define XZB_FILTER_ID_DELTA 0x03u     /* arg = distance 1..256          (delta/delta_encoder.c, delta_decoder.c) */
#define XZB_FILTER_ID_X86 0x04u       /* arg = start offset             (simple/x86.c) */
#define XZB_FILTER_ID_POWERPC 0x05u   /* arg = start offset, 4-aligned  (simple/powerpc.c) */
#define XZB_FILTER_ID_IA64 0x06u      /* arg = start offset, 16-aligned (simple/ia64.c) */
#define XZB_FILTER_ID_ARM 0x07u       /* arg = start offset, 4-aligned  (simple/arm.c) */
#define XZB_FILTER_ID_ARMTHUMB 0x08u  /* arg = start offset, 2-aligned  (simple/armthumb.c) */
#define XZB_FILTER_ID_SPARC 0x09u     /* arg = start offset, 4-aligned  (simple/sparc.c) */
#define XZB_FILTER_ID_ARM64 0x0Au     /* arg = start offset, 4-aligned  (simple/arm64.c) */
#define XZB_FILTER_ID_RISCV 0x0Bu     /* arg = start offset, 2-aligned  (simple/riscv.c) */
typedef struct { uint32_t id, arg; } xzb_filter_spec;
int xzb_ctx_set_filters(xzb_ctx *ctx, const xzb_filter_spec *filters, uint32_t n);
int xzb_get_stats(const xzb_ctx *ctx, xzb_stats *out);

/*
 * ENCODE, device-resident: d_in[0..in_size) (device pointer) is cut into Blocks of block_size
 * bytes (last one may be short), each encoded exactly as worker_encode() does
 * (common/stream_encoder_mt.c:218-359: Block Header with both sizes, LZMA2 data, padding,
 * Check; incompressible fallback :316-344).  The finished Blocks are written back to back to
 * d_out (device pointer, capacity d_out_cap >= nblocks * xzb_block_bound(block_size)).
 * records[i] (host) receives Block i's Index record; *out_size the number of bytes written.
 * No Stream Header/Index/Footer here: see xzb_stream_* and xzb_index_encode().
 */
int xzb_encode_blocks_device(xzb_ctx *ctx, const void *d_in, uint64_t in_size,
		const xzb_lzma_options *opt, uint32_t check, uint64_t block_size,
		void *d_out, uint64_t d_out_cap, uint64_t *out_size, xzb_index_record *records);

/* Same Blocks + records, but `in` and `out` are HOST buffers (copies inside the call).  This is
 * what one rank runs on its shard of Blocks when the Stream is spread over several GPUs. */
int xzb_encode_blocks_host(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		const xzb_lzma_options *opt, uint32_t check, uint64_t block_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size, xzb_index_record *records);

/*
 * ENCODE, host buffers, whole Stream: same bytes as lzma_stream_encoder_mt() +
 * lzma_code(LZMA_FINISH) (stream_encoder_mt.c:716-888, 1027-1208) with lzma_mt.block_size =
 * block_size, lzma_mt.filters = {LZMA2(opt)}, lzma_mt.check = check.
 * Host->device and device->host copies happen inside the call.
 */
int xzb_stream_encode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		const xzb_lzma_options *opt, uint32_t check, uint64_t block_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size);

/*
 * ENCODE, host buffers, one-shot: same bytes as lzma_stream_buffer_encode({LZMA2(opt)}, check, ...)
 * (common/stream_buffer_encoder.c:43-140) and lzma_easy_buffer_encode() (easy_buffer_encoder.c:16-27):
 * ONE Block over the whole input framed as lzma_block_buffer_encode() does
 * (block_buffer_encoder.c:165-325; header sized from lzma2_bound(in_size)), in_size <= 1 GiB.
 * out_cap >= xzb_stream_buffer_bound(in_size) (== lzma_stream_buffer_bound, :17-40) always suffices.
 */
uint64_t xzb_stream_buffer_bound(uint64_t in_size);
/* The Block lzma_block_buffer_encode() produces for zero bytes of input (header, LZMA2 end marker, padding,
 * check of nothing; block_buffer_encoder.c:165-325).  out needs 64 + 32 bytes; returns the size. */
uint32_t xzb_empty_block_encode(uint8_t *out, const xzb_lzma_options *opt, uint32_t check);
int xzb_stream_buffer_encode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		const xzb_lzma_options *opt, uint32_t check,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size);

/*
 * ENCODE, batch of n independent one-shot Streams (liblzma has no such call: this is n lzma_stream_buffer_encode()
 * calls at once).  Item i is in[in_off[i] .. in_off[i] + in_size[i]); its Stream goes to out + out_off[i] (room:
 * out_cap[i]); out_size[i] and ret[i] are what xzb_stream_buffer_encode() gives for that item alone with out_cap[i]
 * -- same bytes, same codes (XZB_BUF_ERROR when it does not fit, XZB_OPTIONS_ERROR above 1 GiB); an item that fails
 * gets out_size[i] = 0 and nothing is written to its slot.  Options, check and the context's Delta/BCJ chain
 * (xzb_ctx_set_filters) apply to every item.  n = 0 and zero-length items are valid (a zero-length item gives the
 * 32-byte Stream with no Block).  The Blocks of all items are coded in waves of similar sizes, side by side on the GPU.
 * The return value is for errors of the whole call (options, check, device).
 */
int xzb_stream_buffer_encode_batch(xzb_ctx *ctx, uint32_t n, const uint8_t *in, const uint64_t *in_off,
		const uint64_t *in_size, const xzb_lzma_options *opt, uint32_t check, uint8_t *out,
		const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint32_t *ret);
/* The same with `in` and `out` in device memory (the offset / size / result arrays stay on the host). */
int xzb_stream_buffer_encode_batch_device(xzb_ctx *ctx, uint32_t n, const uint8_t *in, const uint64_t *in_off,
		const uint64_t *in_size, const xzb_lzma_options *opt, uint32_t check, uint8_t *out,
		const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint32_t *ret);

/* Stream framing around device-encoded Blocks (stream_flags_encoder.c:29-85,
 * index_encoder.c:43-165).  xzb_index_encode(out == NULL) returns the size only. */
uint32_t xzb_stream_header_encode(uint8_t out[12], uint32_t check);
uint32_t xzb_stream_footer_encode(uint8_t out[12], uint32_t check, uint64_t index_size);
uint64_t xzb_index_encode(const xzb_index_record *records, uint64_t count, uint8_t *out);

/*
 * DECODE, host buffers, whole Stream: lzma_stream_decoder(strm, UINT64_MAX, 0) +
 * lzma_code(LZMA_FINISH) (common/stream_decoder.c:101-378, block_decoder.c:64-200,
 * index_hash.c); Blocks whose headers carry both sizes are decoded as one parallel batch
 * (what stream_decoder_mt.c:951-1780 does with threads), others one after another.
 * Only the LZMA2-only filter chain and the None/CRC32/CRC64 checks are in scope.
 */
int xzb_stream_decode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size);
/* Same, and *in_used = bytes of `in` consumed up to and including the Stream Footer (what
 * lzma_stream.total_in would be), for callers that handle LZMA_CONCATENATED streams themselves. */
int xzb_stream_decode_ex(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size, uint64_t *in_used);

/* Decoder flags: XZB_DEC_IGNORE_CHECK is LZMA_IGNORE_CHECK (stream_decoder.c:188-190).  CRC32, CRC64
 * and SHA-256 Check fields are verified; reserved check IDs are skipped as the reference does
 * (block_decoder.c:178-190).  XZB_DEC_SKIP_UNSUPPORTED_CHECK is accepted for compatibility (no effect). */
#define XZB_DEC_SKIP_UNSUPPORTED_CHECK 1u
#define XZB_DEC_IGNORE_CHECK 2u
int xzb_stream_decode_flags(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size, uint64_t *in_used, uint32_t flags);

/* xzb_stream_decode_flags for the LAST part of a Stream whose earlier Blocks were decoded and cut out of `in`
 * by previous calls: `prior` holds their Index records, so the Stream's Index is checked against all of
 * them (the liblzma-named stream decoder uses this to hand over complete Blocks while input still arrives). */
int xzb_stream_decode_prior(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size, uint64_t *in_used, uint32_t flags,
		const xzb_index_record *prior, uint64_t n_prior);

/* Memory the REFERENCE decoder would need for the Blocks of the Stream at `in` (dictionary + 66200 bytes,
 * lzma_raw_decoder_memusage on LP64), walked in order on the host: the first Block above `limit` sets
 * *exceeds, otherwise *memusage is the last Block's figure.  This library keeps nothing of the kind on the
 * host; the number exists so that memlimit / lzma_memusage() callers see the reference's behaviour. */
int xzb_stream_memusage(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size, uint64_t limit, uint64_t *memusage, uint32_t *exceeds);

/* One Stream, result codes as lzma_stream_buffer_decode() maps them
 * (common/stream_buffer_decoder.c:44-88): input that ends early is XZB_DATA_ERROR, an output
 * buffer that is too small is XZB_BUF_ERROR. */
int xzb_stream_buffer_decode(xzb_ctx *ctx, const uint8_t *in, uint64_t in_size,
		uint8_t *out, uint64_t out_cap, uint64_t *out_size, uint64_t *in_used, uint32_t flags);
/* n independent Streams, host buffers: Stream i is in[in_off[i] .. in_off[i] + in_size[i]), its output goes to
 * out + out_off[i] (room: out_cap[i]).  Per item, (ret, out_size, in_used, bytes written) == xzb_stream_buffer_decode()
 * of that item alone with out_cap[i] and `flags`, including bytes delivered before an error.  The Blocks of all
 * Streams are decoded side by side.  The return value is for errors of the whole call (device). */
int xzb_stream_buffer_decode_batch(xzb_ctx *ctx, uint32_t n, const uint8_t *in, const uint64_t *in_off,
		const uint64_t *in_size, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
		uint64_t *out_size, uint64_t *in_used, uint32_t *ret, uint32_t flags);
/* The same with `d_in` and `d_out` in device memory (the offset, size and result arrays stay on the host).  The
 * container (Stream Header, Block Headers, padding, Check fields, Index, Stream Footer) is read on the GPU and each
 * Block decodes straight into its item's slot: no item data crosses PCIe, only per-item results and a few counters.
 *   - Per item, (ret, out_size, in_used) == xzb_stream_buffer_decode_batch() for the same bytes, out_cap and flags
 *     (XZB_DATA_ERROR for input that ends early, XZB_BUF_ERROR for a slot that is too small, XZB_DEC_IGNORE_CHECK),
 *     and bytes [0, out_size[i]) of slot i are its output, those delivered before an error included.
 *   - Nothing outside [out_off[i], out_off[i] + out_cap[i]) is written.  Inside a slot, bytes past out_size[i] may be
 *     written only when ret[i] != XZB_OK (later Blocks of a failed Stream may already have been decoded there).
 *   - n = 0, zero-length items and unaligned offsets are valid.
 * The return value is for errors of the whole call (device, memory). */
int xzb_stream_buffer_decode_batch_device(xzb_ctx *ctx, uint32_t n, const uint8_t *d_in, const uint64_t *in_off,
		const uint64_t *in_size, uint8_t *d_out, const uint64_t *out_off, const uint64_t *out_cap,
		uint64_t *out_size, uint64_t *in_used, uint32_t *ret, uint32_t flags);

/*
 * DECODE, device-resident Blocks: comp_off[i]/comp_size[i] locate Block i's LZMA2 payload
 * (Compressed Data field, without header/padding/check) inside d_in; Block i's output goes to
 * d_out + out_off[i] and must be exactly uncomp_size[i] bytes.  ret[i] receives the per-Block
 * lzma_ret, check_out[i] the CRC (check type `check`) of the decoded bytes.
 * Stands in for worker_decoder(), common/stream_decoder_mt.c:332-496.
 */
int xzb_decode_blocks_device(xzb_ctx *ctx, const void *d_in, const uint64_t *comp_off,
		const uint64_t *comp_size, const uint64_t *uncomp_size, const uint64_t *out_off,
		const uint32_t *dict_size, uint32_t nblocks, uint32_t check, void *d_out,
		uint32_t *ret, uint64_t *check_out);

/* Device memory helpers for callers without a CUDA runtime binding (tests, bench). */
int xzb_device_alloc(xzb_ctx *ctx, void **ptr, uint64_t size);
void xzb_device_free(xzb_ctx *ctx, void *ptr);
int xzb_memcpy_h2d(xzb_ctx *ctx, void *d_dst, const void *h_src, uint64_t size);
int xzb_memcpy_d2h(xzb_ctx *ctx, void *h_dst, const void *d_src, uint64_t size);
const char *xzb_last_error(const xzb_ctx *ctx);
/* Why the last xzb_stream_decode* call on this context returned XZB_BUF_ERROR: 1 = the input ended early,
 * 2 = the output buffer was too small (the two cases of common/stream_buffer_decoder.c:56-71), 0 = neither. */
int xzb_decode_buf_reason(const xzb_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif
