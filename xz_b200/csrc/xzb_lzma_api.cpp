// xzb_lzma_api.cpp -- liblzma's stream-coder entry points (include/xzb200_lzma.h) on top of the
// GPU block path (include/xzb200.h).  Host C++; the state machines mirror common/common.c
// (lzma_code / lzma_end), common/stream_encoder_mt.c (stream_encode_mt: header, blocks in
// order, Index, footer; LZMA_FULL_FLUSH / LZMA_FULL_BARRIER) and common/stream_decoder.c.
// Worker threads become batches ("waves") of Blocks handed to xzb_encode_blocks_host().
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <stdexcept>
#include <thread>
#include <vector>

#include "../../include/xzb200.h"
#include "../../include/xzb200_lzma.h"
#include "xzb_params.h"

namespace {

enum { ISEQ_RUN, ISEQ_SYNC_FLUSH, ISEQ_FULL_FLUSH, ISEQ_FINISH, ISEQ_FULL_BARRIER, ISEQ_END, ISEQ_ERROR };  // common.h:202-211
enum { KIND_ENCODER, KIND_DECODER };

const size_t WAVE_BLOCKS = 64;  // Blocks encoded per GPU batch while streaming
const size_t PART_BLOCKS = 64;  // complete Blocks decoded as a part while the rest of the Stream still arrives

}  // namespace

// ---- the reference's coder seam, common/common.h:222-273 (lzma_next_coder_s) and :291-324 (lzma_internal_s) ----
// lzma_stream.internal has exactly the reference's layout (checked against the reference header by
// tests/test_api_cpu.py), and the GPU stream coders plug into it the way every reference coder does: a `coder`
// object plus the code / end / get_progress / get_check / memconfig / update entries of the vtable.  So the
// lzma_code / lzma_end / lzma_memusage / ... below are generic over the vtable like common.c's, and in a process
// that also holds the reference liblzma (the hybrid `xz` of INTEGRATION.md) either library's lzma_code can drive
// either library's coders, and re-initialising a lzma_stream from one family to the other frees the old coder
// through its own `end` (lzma_next_coder_init, common.h:389-394).
struct xzb_next_coder {
	void *coder;
	lzma_vli id;
	uintptr_t init;
	lzma_ret (*code)(void *coder, const lzma_allocator *allocator, const uint8_t *in, size_t *in_pos, size_t in_size,
			uint8_t *out, size_t *out_pos, size_t out_size, lzma_action action);
	void (*end)(void *coder, const lzma_allocator *allocator);
	void (*get_progress)(void *coder, uint64_t *progress_in, uint64_t *progress_out);
	lzma_check (*get_check)(const void *coder);
	lzma_ret (*memconfig)(void *coder, uint64_t *memusage, uint64_t *old_memlimit, uint64_t new_memlimit);
	lzma_ret (*update)(void *coder, const lzma_allocator *allocator, const lzma_filter *filters, const lzma_filter *reversed_filters);
	lzma_ret (*set_out_limit)(void *coder, uint64_t *uncomp_size, uint64_t out_limit);
};
struct lzma_internal_s {
	xzb_next_coder next;
	unsigned int sequence;              // the ISEQ_* enum
	size_t avail_in;
	bool supported_actions[5];          // LZMA_ACTION_MAX + 1
	bool allow_buf_error;
};
static_assert(sizeof(xzb_next_coder) == 80 && sizeof(lzma_internal_s) == 104, "layout of common/common.h:222-324 (LP64)");

// The coder object behind next.coder for both GPU stream coders.
struct GpuCoder {
	int kind;
	xzb_ctx *ctx;                 // device of the decoder / first device of the encoder (= pool[0])
	std::vector<xzb_ctx *> pool;  // encoder: one context per GPU of this process, created when a wave has work for it
	std::vector<int> devices;     // the CUDA devices the encoder may use
	std::vector<xzb_filter_spec> pre;  // encoder: Delta / BCJ filters in front of LZMA2
	uint64_t progress_in, progress_out;
	std::vector<uint8_t> outq;  // produced, not yet delivered
	size_t outq_pos;
	// encoder
	xzb_lzma_options opt;
	uint32_t check;
	uint64_t block_size;
	std::vector<uint8_t> inbuf;
	std::vector<xzb_index_record> recs;
	bool header_done, tail_done;
	// decoder
	uint32_t flags;
	size_t dec_off;       // start of the first Stream in inbuf that has not been decoded yet
	size_t pad;           // Stream Padding bytes seen since the previous Stream
	bool first_stream, told, finished;
	uint32_t cur_check;   // lzma_get_check()
	uint64_t memlimit, memusage;  // stream_decoder.c:85-90
	std::vector<xzb_index_record> prior;  // records of the current Stream's Blocks that were already decoded and cut out of inbuf
	lzma_ret dec_ret;
	lzma_ret deferred;    // encoder: an option error the reference only reports from lzma_code (BCJ start-offset alignment)
	size_t last_try;      // buffered size at the last speculative decode of a Stream with unsized Blocks (LZMA_RUN)
};

namespace {

void *xalloc(const lzma_allocator *a, size_t size)  // lzma_alloc, common.c:37-52
{
	if (size == 0) size = 1;
	return (a != nullptr && a->alloc != nullptr) ? a->alloc(a->opaque, 1, size) : malloc(size);
}
void xfree(const lzma_allocator *a, void *p)  // lzma_free, common.c:78-87
{
	if (a != nullptr && a->free != nullptr) a->free(a->opaque, p); else free(p);
}

// lzma_next_end, common.c:147-166: works on any coder of either family
void next_end(xzb_next_coder *next, const lzma_allocator *allocator)
{
	if (next->init != (uintptr_t)0) {
		if (next->end != nullptr) next->end(next->coder, allocator);
		else xfree(allocator, next->coder);
		memset(next, 0, sizeof(*next));
		next->id = LZMA_VLI_UNKNOWN;
	}
}

void internal_destroy(lzma_stream *strm)   // lzma_end, common.c:379-389
{
	lzma_internal *si = strm->internal;
	if (si == nullptr) return;
	next_end(&si->next, strm->allocator);
	xfree(strm->allocator, si);
	strm->internal = nullptr;
}

void gpu_coder_end(void *coder, const lzma_allocator *allocator)
{
	GpuCoder *in = static_cast<GpuCoder *>(coder);
	for (xzb_ctx *c : in->pool) if (c) xzb_ctx_destroy(c);
	in->~GpuCoder();
	xfree(allocator, in);
}
void gpu_get_progress(void *coder, uint64_t *progress_in, uint64_t *progress_out)
{
	const GpuCoder *in = static_cast<const GpuCoder *>(coder);
	*progress_in = in->progress_in; *progress_out = in->progress_out;
}

lzma_ret encoder_code(GpuCoder *in, const uint8_t *src, size_t *in_pos, size_t in_size, uint8_t *out, size_t *out_pos, size_t out_size, lzma_action action);
lzma_ret decoder_code(GpuCoder *in, const uint8_t *src, size_t *in_pos, size_t in_size, uint8_t *out, size_t *out_pos, size_t out_size, lzma_action action);
lzma_ret gpu_code(void *coder, const lzma_allocator *, const uint8_t *in, size_t *in_pos, size_t in_size, uint8_t *out, size_t *out_pos,
		size_t out_size, lzma_action action)
{
	GpuCoder *c = static_cast<GpuCoder *>(coder);
	try {   // nothing may unwind through the C ABI (allocation failures of the host queues -> LZMA_MEM_ERROR)
		return c->kind == KIND_ENCODER ? encoder_code(c, in, in_pos, in_size, out, out_pos, out_size, action)
				: decoder_code(c, in, in_pos, in_size, out, out_pos, out_size, action);
	} catch (const std::bad_alloc &) {
		return LZMA_MEM_ERROR;
	} catch (const std::length_error &) {
		return LZMA_MEM_ERROR;
	}
}

// lzma_strm_init (common.c:176-200) + lzma_next_coder_init (common.h:389-394: a coder of another kind -- ours or the
// reference's -- is ended through its own vtable) + the coder object.  `init_marker` identifies the init function.
lzma_ret internal_create(lzma_stream *strm, int kind, uintptr_t init_marker)
{
	if (strm == nullptr) return LZMA_PROG_ERROR;
	if (strm->internal == nullptr) {
		void *mem = xalloc(strm->allocator, sizeof(lzma_internal));
		if (mem == nullptr) return LZMA_MEM_ERROR;
		strm->internal = static_cast<lzma_internal *>(mem);
		memset(&strm->internal->next, 0, sizeof(strm->internal->next));
		strm->internal->next.id = LZMA_VLI_UNKNOWN;
	}
	lzma_internal *si = strm->internal;
	memset(si->supported_actions, 0, sizeof(si->supported_actions));
	si->sequence = ISEQ_RUN;
	si->avail_in = 0;
	si->allow_buf_error = false;
	strm->total_in = 0;
	strm->total_out = 0;
	next_end(&si->next, strm->allocator);   // the GPU coders are always built anew
	void *cm = xalloc(strm->allocator, sizeof(GpuCoder));
	if (cm == nullptr) { internal_destroy(strm); return LZMA_MEM_ERROR; }
	GpuCoder *in = new (cm) GpuCoder();
	si->next.coder = in;
	si->next.init = init_marker;
	si->next.code = &gpu_code;
	si->next.end = &gpu_coder_end;
	si->next.get_progress = &gpu_get_progress;
	in->kind = kind;
	in->ctx = nullptr;
	in->progress_in = in->progress_out = 0;
	in->outq_pos = 0;
	in->header_done = in->tail_done = false;
	in->dec_off = 0; in->pad = 0;
	in->first_stream = true; in->told = false; in->finished = false;
	in->cur_check = 0;
	in->memlimit = UINT64_MAX; in->memusage = 32768;  // LZMA_MEMUSAGE_BASE
	in->dec_ret = LZMA_OK;
	in->deferred = LZMA_OK;
	in->last_try = 0;
	// Devices: XZB_DEVICE=n pins everything to one GPU; otherwise the decoder uses device 0 and the threaded encoder deals
	// the Blocks of a wave over all GPUs of the process (XZB_DEVICES=a,b,c restricts the set) -- the worker fan-out of
	// stream_encoder_mt.c:362-595 / :716-888 behind the one lzma_stream_encoder_mt call.
	const char *dev = getenv("XZB_DEVICE");
	const char *devs = getenv("XZB_DEVICES");
	if (dev) in->devices.push_back(atoi(dev));
	else if (kind == KIND_ENCODER && devs) {
		for (const char *q = devs; *q;) { in->devices.push_back(atoi(q)); while (*q && *q != ',') ++q; if (*q == ',') ++q; }
	} else if (kind == KIND_ENCODER) {
		const int n = xzb_device_count();
		for (int i = 0; i < n; ++i) in->devices.push_back(i);
	}
	if (in->devices.empty()) in->devices.push_back(0);
	const int r = xzb_ctx_create(&in->ctx, in->devices[0]);
	if (r != 0) { internal_destroy(strm); return (lzma_ret)r; }
	in->pool.push_back(in->ctx);
	return LZMA_OK;
}

bool to_xzb_options(const lzma_options_lzma *o, xzb_lzma_options *x)
{
	if (o->preset_dict != nullptr && o->preset_dict_size > 0) return false;  // preset dictionaries: SURVEY 8(f) rank 3
	x->dict_size = o->dict_size; x->lc = o->lc; x->lp = o->lp; x->pb = o->pb;
	x->mode = (uint32_t)o->mode; x->nice_len = o->nice_len; x->mf = (uint32_t)o->mf; x->depth = o->depth;
	return true;
}

void deliver(GpuCoder *in, uint8_t *out, size_t *out_pos, size_t out_size)
{
	const size_t n = std::min(in->outq.size() - in->outq_pos, out_size - *out_pos);
	if (n) { memcpy(out + *out_pos, in->outq.data() + in->outq_pos, n); in->outq_pos += n; *out_pos += n; }
	if (in->outq_pos == in->outq.size()) { in->outq.clear(); in->outq_pos = 0; }
}

// Encode the first `bytes` of inbuf as Blocks and queue them.
lzma_ret encode_prefix(GpuCoder *in, size_t bytes)
{
	if (bytes == 0) return LZMA_OK;
	const uint64_t nblocks = (bytes + in->block_size - 1) / in->block_size;
	const size_t cap = (size_t)(nblocks * xzb_block_bound(in->block_size));
	const size_t at = in->outq.size();
	in->outq.resize(at + cap);
	std::vector<xzb_index_record> recs(nblocks);
	uint64_t produced = 0;
	int r = 0;
	const size_t nd = (size_t)std::min<uint64_t>(in->devices.size(), nblocks);
	if (nd <= 1) {
		r = xzb_encode_blocks_host(in->ctx, in->inbuf.data(), bytes, &in->opt, in->check, in->block_size,
				in->outq.data() + at, cap, &produced, recs.data());
	} else {
		// Blocks [first_d, first_{d+1}) go to GPU d, one host thread per GPU (each call binds its thread to its device);
		// the finished Blocks are packed together in Block order afterwards.  Nothing is exchanged between the GPUs.
		while (in->pool.size() < nd) {
			xzb_ctx *c = nullptr;
			int rc = xzb_ctx_create(&c, in->devices[in->pool.size()]);
			if (rc == 0) { in->pool.push_back(c); rc = xzb_ctx_set_filters(c, in->pre.data(), (uint32_t)in->pre.size()); }
			if (rc != 0) { in->outq.resize(at); return (lzma_ret)rc; }
		}
		const uint64_t bound = xzb_block_bound(in->block_size);
		std::vector<uint64_t> first(nd + 1), got(nd, 0);
		std::vector<int> rr(nd, 0);
		for (size_t d = 0; d <= nd; ++d) first[d] = nblocks * d / nd;
		std::vector<std::thread> th;
		for (size_t d = 0; d < nd; ++d) {
			th.emplace_back([&, d]() {
				const uint64_t off = first[d] * in->block_size;
				const uint64_t len = std::min<uint64_t>(bytes, first[d + 1] * in->block_size) - off;
				rr[d] = xzb_encode_blocks_host(in->pool[d], in->inbuf.data() + off, len, &in->opt, in->check, in->block_size,
						in->outq.data() + at + first[d] * bound, (first[d + 1] - first[d]) * bound, &got[d], recs.data() + first[d]);
			});
		}
		for (auto &t : th) t.join();
		for (size_t d = 0; d < nd; ++d) {
			if (rr[d] != 0 && r == 0) r = rr[d];
			if (r == 0) {
				if (d != 0) memmove(in->outq.data() + at + produced, in->outq.data() + at + first[d] * bound, (size_t)got[d]);
				produced += got[d];
			}
		}
	}
	if (r != 0) { in->outq.resize(at); return (lzma_ret)r; }
	in->outq.resize(at + produced);
	in->recs.insert(in->recs.end(), recs.begin(), recs.end());
	in->inbuf.erase(in->inbuf.begin(), in->inbuf.begin() + bytes);
	in->progress_in += bytes;
	in->progress_out += produced;
	return LZMA_OK;
}

// stream_encode_mt, common/stream_encoder_mt.c:716-888
lzma_ret encoder_code(GpuCoder *in, const uint8_t *src, size_t *in_pos, size_t in_size, uint8_t *out, size_t *out_pos,
		size_t out_size, lzma_action action)
{
	if (!in->header_done) {  // SEQ_STREAM_HEADER
		uint8_t hdr[12];
		xzb_stream_header_encode(hdr, in->check);
		in->outq.insert(in->outq.end(), hdr, hdr + 12);
		in->header_done = true;
	}
	deliver(in, out, out_pos, out_size);
	if (in->deferred != LZMA_OK) {   // the worker's coder set-up failed: Stream Header out, input taken, then the error (like the reference)
		*in_pos = in_size;
		return in->deferred;
	}
	// SEQ_BLOCK: take all the input (stream_encode_in copies it into the worker buffers, :598-661)
	if (*in_pos < in_size) {
		in->inbuf.insert(in->inbuf.end(), src + *in_pos, src + in_size);
		*in_pos = in_size;
	}
	const size_t wave = (size_t)(WAVE_BLOCKS * in->block_size);
	while (in->inbuf.size() >= wave) {
		const lzma_ret r = encode_prefix(in, wave);
		if (r != LZMA_OK) return r;
	}
	if (action == LZMA_RUN) { deliver(in, out, out_pos, out_size); return LZMA_OK; }
	// LZMA_FINISH / LZMA_FULL_FLUSH / LZMA_FULL_BARRIER: the pending partial Block ends here (:617-624)
	if (!in->inbuf.empty()) {
		const lzma_ret r = encode_prefix(in, in->inbuf.size());
		if (r != LZMA_OK) return r;
	}
	if (action == LZMA_FULL_BARRIER) { deliver(in, out, out_pos, out_size); return LZMA_STREAM_END; }
	if (action == LZMA_FINISH && !in->tail_done) {  // SEQ_INDEX + SEQ_STREAM_FOOTER :842-883
		const uint64_t isz = xzb_index_encode(in->recs.data(), in->recs.size(), nullptr);
		const size_t at = in->outq.size();
		in->outq.resize(at + isz + 12);
		xzb_index_encode(in->recs.data(), in->recs.size(), in->outq.data() + at);
		xzb_stream_footer_encode(in->outq.data() + at + isz, in->check, isz);
		in->progress_out += isz + 12;
		in->tail_done = true;
	}
	deliver(in, out, out_pos, out_size);
	return in->outq.empty() ? LZMA_STREAM_END : LZMA_OK;
}

const uint32_t *crc32_table()  // for the container readers of xzb_frame.cuh
{
	static const XzbHostTables t = [] { XzbHostTables h; xzb_make_tables(&h); return h; }();
	return t.crc32;
}

// Is a whole Stream (header .. footer) buffered?  Walks sized Block Headers only; unsized Blocks
// (single-threaded encoders) are only known to be complete at LZMA_FINISH.  Lax on purpose (the decoder validates):
// a Compressed Size counts as far as it goes unless it has no last byte within nine.
bool stream_complete(const std::vector<uint8_t> &b, size_t *end)
{
	if (b.size() < 12) return false;
	const uint32_t csize = xzb_check_field_size(b[7] & 0x0F);
	size_t ip = 12;
	for (;;) {
		if (ip >= b.size()) return false;
		if (b[ip] == 0x00) break;
		XzbBlockFraming f;
		if (!xzb_block_framing(b.data() + ip, b.size() - ip, &f) || !(f.flags & 0x40) || f.comp.st == XZB_VLI_LONG) return false;
		const uint64_t total = f.hsize + ((f.comp.v + 3) & ~3ull) + csize;
		if (b.size() - ip < total) return false;
		ip += (size_t)total;
	}
	XzbIndexRead x;
	xzb_index_read(crc32_table(), b.data() + ip, b.size() - ip, nullptr, &x);
	if (!x.listed || b.size() - ip < x.end + 12) return false;
	*end = ip + (size_t)x.end + 12;
	return true;
}

// No LZMA2 payload expands by more than this factor: the cheapest symbol, a rep0 match of 273 bytes, still costs
// 14 binary decisions of at least log2(2048 / 2017) bits each (probabilities saturate at 31/2048), ~7000 : 1.
const uint64_t MAX_RATIO = 8192;

// First guess of a Stream's uncompressed size from its Block Headers.  Header fields come from untrusted input, so a
// claimed size counts only as far as the compressed bytes can justify it; unsized Blocks start from a modest guess and
// the caller grows the buffer when the decoder reports that the output did not fit.  Walks as stream_complete did.
uint64_t stream_out_bound(const std::vector<uint8_t> &b, size_t off, size_t len, bool complete)
{
	if (!complete) return (uint64_t)len * 16 + (1u << 20);
	uint64_t cap = 0;
	size_t ip = off + 12;
	const uint32_t csize = xzb_check_field_size(b[off + 7] & 0x0F);
	while (b[ip] != 0x00) {
		XzbBlockFraming f;
		xzb_block_framing(b.data() + ip, b.size() - ip, &f);
		uint64_t unc = (f.flags & 0x80) ? f.uncomp.v : f.comp.v * 16 + 65536;
		if (unc > f.comp.v * MAX_RATIO + 65536) unc = f.comp.v * MAX_RATIO + 65536;
		cap += unc;
		ip += f.hsize + (size_t)((f.comp.v + 3) & ~3ull) + csize;
	}
	return cap;
}

// Complete sized Blocks at the front of an incomplete Stream (b = Stream Header + Blocks so far): how many,
// where they end, their uncompressed total, and their Index records as the headers state them.  Lax like
// stream_complete, except that the Compressed Size must end inside the header, before the Uncompressed Size.
static size_t complete_blocks(const std::vector<uint8_t> &b, size_t *end, uint64_t *unc_total, std::vector<xzb_index_record> *recs)
{
	size_t n = 0, ip = 12;
	*end = 12; *unc_total = 0;
	if (b.size() < 12) return 0;
	const size_t csize = xzb_check_field_size(b[7] & 0x0F);
	while (ip < b.size() && b[ip] != 0x00) {
		XzbBlockFraming f;
		if (!xzb_block_framing(b.data() + ip, b.size() - ip, &f) || (f.flags & 0xC0) != 0xC0) break;  // both sizes must be in the header
		const uint64_t comp = f.comp.v, unc = f.uncomp.v;
		if (f.comp.st == XZB_VLI_LONG || f.comp.end >= f.hsize || f.uncomp.st == XZB_VLI_LONG) break;
		if (comp == 0 || comp > (1ull << 40) || unc > comp * MAX_RATIO + 65536) break;  // a size the payload cannot justify is left to the final pass
		const uint64_t total = f.hsize + ((comp + 3) & ~3ull) + csize;
		if (b.size() - ip < total) break;
		ip += (size_t)total;
		*unc_total += unc;
		recs->push_back(xzb_index_record{ f.hsize + comp + csize, unc });
		++n; *end = ip;
	}
	return n;
}

static uint32_t dec_flags(uint32_t lzma_flags)
{
	return (lzma_flags & LZMA_IGNORE_CHECK) ? XZB_DEC_IGNORE_CHECK : 0u;
}

// Check ID of a valid Stream Header at p (12 bytes), or -1.
static int header_check_id(const uint8_t *p)
{
	uint32_t check = 0;
	return xzb_stream_header_decode(crc32_table(), p, &check) == XZB_OK ? (int)check : -1;
}

// Do the buffered bytes end in a valid Stream Footer (stream_flags_decoder.c:51-83)?  Used under LZMA_RUN to notice
// the end of a Stream whose Blocks carry no sizes (single-threaded encoders): only then is a decode attempted.
static bool footer_at_end(const std::vector<uint8_t> &b)
{
	if (b.size() < 32 || (b.size() & 3) != 0) return false;
	uint32_t check = 0; uint64_t index_size = 0;
	return xzb_stream_footer_decode(crc32_table(), b.data() + b.size() - 12, &check, &index_size) == XZB_OK;
}

// stream_decode, common/stream_decoder.c:101-378, as a resumable loop over the buffered input: a
// Stream is decoded as one GPU batch as soon as it is completely buffered (or at LZMA_FINISH).
// LZMA_TELL_* codes are returned once per Stream right after its header (:139-151).  With
// LZMA_CONCATENATED (:334-371) Stream Padding must be a multiple of four zero bytes and the
// decoder only finishes at LZMA_FINISH.
lzma_ret decoder_code(GpuCoder *in, const uint8_t *src, size_t *in_pos, size_t in_size, uint8_t *out, size_t *out_pos,
		size_t out_size, lzma_action action)
{
	if (*in_pos < in_size && !in->finished) {
		in->inbuf.insert(in->inbuf.end(), src + *in_pos, src + in_size);
		in->progress_in += in_size - *in_pos;
		*in_pos = in_size;
	}
	const bool concatenated = (in->flags & LZMA_CONCATENATED) != 0;
	for (;;) {
		deliver(in, out, out_pos, out_size);
		if (!in->outq.empty()) return LZMA_OK;
		if (in->finished) return in->dec_ret;
		if (!in->first_stream) {  // SEQ_STREAM_PADDING :337-371
			while (in->dec_off < in->inbuf.size() && in->inbuf[in->dec_off] == 0x00) { ++in->dec_off; ++in->pad; }
			if (in->dec_off >= in->inbuf.size()) {
				if (action != LZMA_FINISH) return LZMA_OK;
				in->finished = true;
				in->dec_ret = (in->pad & 3) == 0 ? LZMA_STREAM_END : LZMA_DATA_ERROR;
				continue;
			}
			if (in->pad & 3) { in->finished = true; in->dec_ret = LZMA_DATA_ERROR; continue; }
		}
		const size_t avail = in->inbuf.size() - in->dec_off;
		if (!in->told && avail >= 12) {
			in->told = true;
			const int chk = header_check_id(in->inbuf.data() + in->dec_off);
			if (chk >= 0) {
				in->cur_check = (uint32_t)chk;
				if ((in->flags & LZMA_TELL_NO_CHECK) && chk == 0) return LZMA_NO_CHECK;
				if ((in->flags & LZMA_TELL_UNSUPPORTED_CHECK) && !lzma_check_is_supported((lzma_check)chk)) return LZMA_UNSUPPORTED_CHECK;
				if (in->flags & LZMA_TELL_ANY_CHECK) return LZMA_GET_CHECK;
			}
		}
		// the not yet decoded rest of the input as its own buffer for the bound helpers
		std::vector<uint8_t> rest;
		const std::vector<uint8_t> *view = &in->inbuf;
		if (in->dec_off != 0) { rest.assign(in->inbuf.begin() + in->dec_off, in->inbuf.end()); view = &rest; }
		size_t end = 0;
		const bool complete = stream_complete(*view, &end);
		bool speculative = false;
		if (!complete && action != LZMA_FINISH) {
			// Progressive output: once PART_BLOCKS complete Blocks are waiting they are decoded as a part (wrapped
			// with an Index + Footer made from their own headers, so the one-shot decoder validates each Block
			// exactly as it would inside the whole Stream) and cut out of the buffer; their records go to
			// `prior` for the check of the real Index at the end.
			size_t bend = 0; uint64_t unc = 0;
			std::vector<xzb_index_record> recs(in->prior);
			const size_t nb = complete_blocks(*view, &bend, &unc, &recs);
			if (nb < PART_BLOCKS) {
				// Unsized Blocks hide the end of the Stream; the reference's decoder returns LZMA_STREAM_END under LZMA_RUN
				// once the footer is in (stream_decoder.c:309-331).  When the buffered bytes end in a valid Stream Footer
				// the whole buffer is decoded; "input ended early" from that attempt just means: not yet.
				if (view->size() != in->last_try && footer_at_end(*view)) {
					in->last_try = view->size();
					speculative = true;
				} else {
					return LZMA_OK;
				}
			}
			if (!speculative) {
			uint64_t mu = 0; uint32_t exceeds = 0;
			xzb_stream_memusage(in->ctx, view->data(), bend, in->memlimit, &mu, &exceeds);
			in->memusage = mu;
			if (exceeds) return LZMA_MEMLIMIT_ERROR;
			const uint64_t isz = xzb_index_encode(recs.data(), recs.size(), nullptr);
			std::vector<uint8_t> part(bend + (size_t)isz + 12);
			memcpy(part.data(), view->data(), bend);
			xzb_index_encode(recs.data(), recs.size(), part.data() + bend);
			xzb_stream_footer_encode(part.data() + bend + isz, in->cur_check, isz);
			const size_t at = in->outq.size();
			in->outq.resize(at + (size_t)unc + 1);
			uint64_t produced = 0, used = 0;
			int r = xzb_stream_decode_prior(in->ctx, part.data(), part.size(), in->outq.data() + at, unc, &produced, &used, dec_flags(in->flags),
					in->prior.data(), in->prior.size());
			in->outq.resize(at + (size_t)produced);
			in->progress_out += produced;
			if (r != 0) { in->finished = true; in->dec_ret = (lzma_ret)r; continue; }
			in->prior.swap(recs);
			in->inbuf.erase(in->inbuf.begin() + in->dec_off + 12, in->inbuf.begin() + in->dec_off + bend);
			continue;
			}
		}
		{  // SEQ_BLOCK_INIT memory limit, stream_decoder.c:199-232 (recoverable: lzma_memlimit_set + lzma_code again)
			uint64_t mu = 0; uint32_t exceeds = 0;
			xzb_stream_memusage(in->ctx, view->data(), view->size(), in->memlimit, &mu, &exceeds);
			if (view->size() > 12 && (*view)[12] != 0x00) in->memusage = mu;
			if (exceeds) return LZMA_MEMLIMIT_ERROR;
		}
		uint64_t cap = stream_out_bound(*view, 0, view->size(), complete);
		const uint64_t cap_max = (uint64_t)view->size() * MAX_RATIO + 65536;
		const size_t at = in->outq.size();
		uint64_t produced = 0, used = 0;
		int r;
		for (;;) {
			in->outq.resize(at + (size_t)cap + 1);
			produced = 0; used = 0;
			r = xzb_stream_decode_prior(in->ctx, view->data(), complete ? end : view->size(), in->outq.data() + at, cap, &produced, &used,
					dec_flags(in->flags), in->prior.data(), in->prior.size());
			// XZB_BUF_ERROR has two meanings (xzb_decode_buf_reason): 2 = the output buffer was too small for a Block without
			// an Uncompressed Size (ratios go into the thousands) -> grow and decode again; 1 = the input ended early.
			if (r == 10 && xzb_decode_buf_reason(in->ctx) == 2 && cap < cap_max) {
				cap = cap * 8 < cap_max ? cap * 8 : cap_max;
				continue;
			}
			break;
		}
		if (speculative && r == 10 && xzb_decode_buf_reason(in->ctx) != 2) {   // the Stream is not complete yet after all
			in->outq.resize(at);
			return LZMA_OK;
		}
		in->outq.resize(at + (size_t)produced);
		in->progress_out += produced;
		if (r == 7 && !in->first_stream) r = 9;  // LZMA_FORMAT_ERROR in a later Stream is LZMA_DATA_ERROR (stream_decoder.c:121-123)
		if (r != 0) {
			// LZMA_BUF_ERROR from the one-shot decoder means "input ended early": with lzma_code that is
			// LZMA_OK now and LZMA_BUF_ERROR on the next call without progress (common.c:316-330)
			in->finished = true;
			in->dec_ret = r == 10 ? LZMA_OK : (lzma_ret)r;
			continue;
		}
		in->dec_off += (size_t)used;
		in->prior.clear();
		in->first_stream = false; in->told = false; in->pad = 0;
		if (!concatenated) { in->finished = true; in->dec_ret = LZMA_STREAM_END; }
	}
}

}  // namespace

extern "C" {

lzma_bool lzma_lzma_preset(lzma_options_lzma *options, uint32_t preset)
{
	xzb_lzma_options x;
	if (xzb_lzma_preset(&x, preset) != 0) return 1;
	options->preset_dict = nullptr; options->preset_dict_size = 0;
	options->dict_size = x.dict_size; options->lc = x.lc; options->lp = x.lp; options->pb = x.pb;
	options->mode = (lzma_mode)x.mode; options->nice_len = x.nice_len; options->mf = (lzma_match_finder)x.mf; options->depth = x.depth;
	return 0;
}

lzma_bool lzma_check_is_supported(lzma_check check)
{
	return check == LZMA_CHECK_NONE || check == LZMA_CHECK_CRC32 || check == LZMA_CHECK_CRC64 || check == LZMA_CHECK_SHA256;
}
uint32_t lzma_check_size(lzma_check check)
{
	return xzb_check_field_size((uint32_t)check);
}
size_t lzma_block_buffer_bound(size_t uncompressed_size) { return (size_t)xzb_block_bound(uncompressed_size); }

// ---- one-shot buffer API ----
// The one-shot calls have no lzma_stream to hang a context on: they share one lazily created
// context per process, serialised by a mutex (a context owns one CUDA stream and workspace).
static std::mutex g_oneshot_mu;
static xzb_ctx *g_oneshot_ctx = nullptr;
static lzma_ret oneshot_ctx(xzb_ctx **out)
{
	if (g_oneshot_ctx == nullptr) {
		const char *dev = getenv("XZB_DEVICE");
		const int r = xzb_ctx_create(&g_oneshot_ctx, dev ? atoi(dev) : 0);
		if (r != 0) { g_oneshot_ctx = nullptr; return (lzma_ret)r; }
	}
	*out = g_oneshot_ctx;
	return LZMA_OK;
}

static bool valid_lzma2_options(const xzb_lzma_options &x)
{
	return !(x.lc > 4 || x.lp > 4 || x.lc + x.lp > 4 || x.pb > 4 || x.nice_len < 2 || x.nice_len > 273
			|| (x.mode != 1 && x.mode != 2) || x.dict_size < 4096 || x.dict_size > (1u << 30) + (1u << 29)
			|| (x.mf != 0x03 && x.mf != 0x04 && x.mf != 0x12 && x.mf != 0x13 && x.mf != 0x14));
}

size_t lzma_stream_buffer_bound(size_t uncompressed_size) { return (size_t)xzb_stream_buffer_bound(uncompressed_size); }

// common/stream_buffer_encoder.c:43-140
lzma_ret lzma_stream_buffer_encode(lzma_filter *filters, lzma_check check, const lzma_allocator *allocator,
		const uint8_t *in, size_t in_size, uint8_t *out, size_t *out_pos_ptr, size_t out_size)
{
	(void)allocator;
	if (filters == nullptr || (unsigned)check > 15 || (in == nullptr && in_size != 0) || out == nullptr
			|| out_pos_ptr == nullptr || *out_pos_ptr > out_size)
		return LZMA_PROG_ERROR;
	if (!lzma_check_is_supported(check)) return LZMA_UNSUPPORTED_CHECK;
	if (out_size - *out_pos_ptr <= 2 * 12) return LZMA_BUF_ERROR;
	xzb_lzma_options x;
	if (filters[0].id != LZMA_FILTER_LZMA2 || filters[1].id != LZMA_VLI_UNKNOWN || filters[0].options == nullptr) return LZMA_OPTIONS_ERROR;
	if (!to_xzb_options((const lzma_options_lzma *)filters[0].options, &x) || !valid_lzma2_options(x)) return LZMA_OPTIONS_ERROR;
	if (in_size > ((size_t)1 << 30)) return LZMA_OPTIONS_ERROR;  // GPU path limit (DESIGN.md)
	std::lock_guard<std::mutex> lock(g_oneshot_mu);
	xzb_ctx *ctx = nullptr;
	const lzma_ret rc = oneshot_ctx(&ctx);
	if (rc != LZMA_OK) return rc;
	// The reference stops as soon as `out` is full; here the Stream is produced whole and handed
	// over only when it fits, which is the same observable result (LZMA_BUF_ERROR, *out_pos kept).
	const size_t room = out_size - *out_pos_ptr;
	const size_t bound = (size_t)xzb_stream_buffer_bound(in_size);
	uint64_t produced = 0;
	if (room >= bound) {
		const int r = xzb_stream_buffer_encode(ctx, in, in_size, &x, (uint32_t)check, out + *out_pos_ptr, room, &produced);
		if (r != 0) return (lzma_ret)r;
	} else {
		std::vector<uint8_t> tmp(bound);
		const int r = xzb_stream_buffer_encode(ctx, in, in_size, &x, (uint32_t)check, tmp.data(), bound, &produced);
		if (r != 0) return (lzma_ret)r;
		if (produced > room) return LZMA_BUF_ERROR;
		memcpy(out + *out_pos_ptr, tmp.data(), (size_t)produced);
	}
	*out_pos_ptr += (size_t)produced;
	return LZMA_OK;
}

// common/block_buffer_encoder.c:213-325
lzma_ret lzma_block_buffer_encode(lzma_block *block, const lzma_allocator *allocator,
		const uint8_t *in, size_t in_size, uint8_t *out, size_t *out_pos, size_t out_size)
{
	(void)allocator;
	if (block == nullptr || (in == nullptr && in_size != 0) || out == nullptr || out_pos == nullptr || *out_pos > out_size) return LZMA_PROG_ERROR;
	if (block->version > 1) return LZMA_OPTIONS_ERROR;
	if ((unsigned)block->check > 15 || block->filters == nullptr) return LZMA_PROG_ERROR;
	if (!lzma_check_is_supported(block->check)) return LZMA_UNSUPPORTED_CHECK;
	size_t room = out_size - *out_pos;
	room -= room & 3;  // a Block is a multiple of four bytes (:233-236)
	const size_t check_size = lzma_check_size(block->check);
	if (room <= check_size) return LZMA_BUF_ERROR;
	const lzma_filter *f = block->filters;
	xzb_lzma_options x;
	if (f[0].id != LZMA_FILTER_LZMA2 || f[1].id != LZMA_VLI_UNKNOWN || f[0].options == nullptr) return LZMA_OPTIONS_ERROR;
	if (!to_xzb_options((const lzma_options_lzma *)f[0].options, &x) || !valid_lzma2_options(x)) return LZMA_OPTIONS_ERROR;
	if (in_size > ((size_t)1 << 30)) return LZMA_OPTIONS_ERROR;  // GPU path limit (DESIGN.md)
	std::vector<uint8_t> tmp;
	size_t at = 0;  // the Block in tmp
	if (in_size == 0) {
		// nothing to search or code: header + the LZMA2 end marker alone (lzma2_encoder.c:141-150)
		tmp.resize(64 + check_size);
		tmp.resize(xzb_empty_block_encode(tmp.data(), &x, (uint32_t)block->check));
	} else {
		std::lock_guard<std::mutex> lock(g_oneshot_mu);
		xzb_ctx *ctx = nullptr;
		const lzma_ret rc = oneshot_ctx(&ctx);
		if (rc != LZMA_OK) return rc;
		const size_t bound = (size_t)xzb_stream_buffer_bound(in_size);
		tmp.resize(bound);
		uint64_t produced = 0;
		const int r = xzb_stream_buffer_encode(ctx, in, in_size, &x, (uint32_t)block->check, tmp.data(), bound, &produced);
		if (r != 0) return (lzma_ret)r;
		at = 12;
	}
	const uint8_t *blk = tmp.data() + at;
	XzbBlockFraming hdr;  // a header this library wrote: both sizes are in it
	xzb_block_framing(blk, tmp.size() - at, &hdr);
	const size_t total = hdr.hsize + (size_t)((hdr.comp.v + 3) & ~3ull) + check_size;
	if (total > room) return LZMA_BUF_ERROR;
	memcpy(out + *out_pos, blk, total);
	*out_pos += total;
	block->header_size = hdr.hsize;
	block->compressed_size = hdr.comp.v;
	block->uncompressed_size = in_size;
	memcpy(block->raw_check, blk + total - check_size, check_size);
	return LZMA_OK;
}

// common/easy_buffer_encoder.c:16-27
lzma_ret lzma_easy_buffer_encode(uint32_t preset, lzma_check check, const lzma_allocator *allocator,
		const uint8_t *in, size_t in_size, uint8_t *out, size_t *out_pos, size_t out_size)
{
	lzma_options_lzma o;
	if (lzma_lzma_preset(&o, preset)) return LZMA_OPTIONS_ERROR;
	lzma_filter f[2] = { { LZMA_FILTER_LZMA2, &o }, { LZMA_VLI_UNKNOWN, nullptr } };
	return lzma_stream_buffer_encode(f, check, allocator, in, in_size, out, out_pos, out_size);
}

// common/stream_buffer_decoder.c:14-92
lzma_ret lzma_stream_buffer_decode(uint64_t *memlimit, uint32_t flags, const lzma_allocator *allocator,
		const uint8_t *in, size_t *in_pos, size_t in_size, uint8_t *out, size_t *out_pos, size_t out_size)
{
	(void)allocator; (void)memlimit;
	if (in_pos == nullptr || (in == nullptr && *in_pos != in_size) || *in_pos > in_size || out_pos == nullptr
			|| (out == nullptr && *out_pos != out_size) || *out_pos > out_size)
		return LZMA_PROG_ERROR;
	if (flags & LZMA_TELL_ANY_CHECK) return LZMA_PROG_ERROR;
	if (flags & ~(LZMA_TELL_NO_CHECK | LZMA_TELL_UNSUPPORTED_CHECK | LZMA_TELL_ANY_CHECK | LZMA_CONCATENATED | LZMA_IGNORE_CHECK | LZMA_FAIL_FAST))
		return LZMA_OPTIONS_ERROR;
	std::lock_guard<std::mutex> lock(g_oneshot_mu);
	xzb_ctx *ctx = nullptr;
	const lzma_ret rc = oneshot_ctx(&ctx);
	if (rc != LZMA_OK) return rc;
	size_t ip = *in_pos, op = *out_pos;
	bool first = true;
	static uint8_t dummy_out[1];
	for (;;) {
		// LZMA_TELL_NO_CHECK / LZMA_TELL_UNSUPPORTED_CHECK after a valid Stream Header
		// (stream_decoder.c:139-151): the code is not LZMA_STREAM_END, so the one-shot call fails with it
		const int chk = in_size - ip >= 12 ? header_check_id(in + ip) : -1;
		if ((flags & LZMA_TELL_NO_CHECK) && chk == 0) return LZMA_NO_CHECK;
		if ((flags & LZMA_TELL_UNSUPPORTED_CHECK) && chk >= 0 && !lzma_check_is_supported((lzma_check)chk)) return LZMA_UNSUPPORTED_CHECK;
		uint64_t produced = 0, used = 0;
		int r = xzb_stream_buffer_decode(ctx, in + ip, in_size - ip, out ? out + op : dummy_out, out_size - op, &produced, &used, dec_flags(flags));
		if (r == 7 && !first) r = 9;  // LZMA_FORMAT_ERROR in a later Stream is LZMA_DATA_ERROR (stream_decoder.c:121-123)
		if (r != 0) return (lzma_ret)r;
		ip += (size_t)used; op += (size_t)produced;
		first = false;
		if (!(flags & LZMA_CONCATENATED)) break;
		size_t pad = 0;  // SEQ_STREAM_PADDING, stream_decoder.c:337-371
		while (ip < in_size && in[ip] == 0x00) { ++ip; ++pad; }
		if (pad & 3) return LZMA_DATA_ERROR;
		if (ip >= in_size) break;
	}
	*in_pos = ip; *out_pos = op;
	return LZMA_OK;
}

// get_options, common/stream_encoder_mt.c:955-1000
// A filter chain of the table common/filter_encoder.c:59-182 as this path takes it: up to three Delta / BCJ filters,
// LZMA2 last (validate_chain, filter_common.c:122-249).  `pre` receives the filters in front of LZMA2.
static lzma_ret parse_chain(const lzma_filter *f, xzb_lzma_options *x, std::vector<xzb_filter_spec> *pre)
{
	if (f == nullptr || f[0].id == LZMA_VLI_UNKNOWN) return LZMA_OPTIONS_ERROR;
	size_t n = 0;
	while (f[n].id != LZMA_VLI_UNKNOWN) { if (++n > 4) return LZMA_OPTIONS_ERROR; }
	if (f[n - 1].id != LZMA_FILTER_LZMA2 || f[n - 1].options == nullptr) return LZMA_OPTIONS_ERROR;
	if (!to_xzb_options((const lzma_options_lzma *)f[n - 1].options, x)) return LZMA_OPTIONS_ERROR;
	for (size_t i = 0; i + 1 < n; ++i) {
		xzb_filter_spec s;
		s.id = (uint32_t)f[i].id; s.arg = 0;
		if (f[i].id == LZMA_FILTER_DELTA) {
			const lzma_options_delta *od = (const lzma_options_delta *)f[i].options;
			if (od == nullptr || od->type != LZMA_DELTA_TYPE_BYTE || od->dist < 1 || od->dist > 256) return LZMA_OPTIONS_ERROR;
			s.arg = od->dist;
		} else if (f[i].id >= LZMA_FILTER_X86 && f[i].id <= LZMA_FILTER_RISCV) {
			const lzma_options_bcj *ob = (const lzma_options_bcj *)f[i].options;
			s.arg = ob ? ob->start_offset : 0;   // (its alignment is only checked when a Block's coder is set up, see below)
		} else {
			return LZMA_OPTIONS_ERROR;   // LZMA2 anywhere but last, unknown IDs
		}
		if (pre) pre->push_back(s);
	}
	return LZMA_OK;
}

static lzma_ret get_options(const lzma_mt *options, xzb_lzma_options *x, uint64_t *block_size, std::vector<xzb_filter_spec> *pre = nullptr)
{
	if (options == nullptr) return LZMA_PROG_ERROR;
	if (options->flags != 0 || options->threads == 0 || options->threads > 16384) return LZMA_OPTIONS_ERROR;
	if (options->filters != nullptr) {
		const lzma_ret rc = parse_chain(options->filters, x, pre);
		if (rc != LZMA_OK) return rc;
	} else {
		if (xzb_lzma_preset(x, options->preset) != 0) return LZMA_OPTIONS_ERROR;
	}
	if (options->block_size > 0) {
		if (options->block_size > UINT64_MAX / 16384) return LZMA_OPTIONS_ERROR;  // BLOCK_SIZE_MAX, :24-30
		*block_size = options->block_size;
	} else {
		*block_size = (uint64_t)x->dict_size * 3 > (1u << 20) ? (uint64_t)x->dict_size * 3 : (1u << 20);  // lzma_lzma2_block_size
	}
	return LZMA_OK;
}

uint64_t lzma_mt_block_size(const lzma_filter *filters)
{
	// filter_encoder.c:262-283: the largest block_size() of the chain; only LZMA2 has one (lzma2_encoder.c:403-413)
	if (filters == nullptr) return UINT64_MAX;
	uint64_t best = 0;
	for (size_t i = 0; filters[i].id != LZMA_VLI_UNKNOWN; ++i) {
		if (i >= 4) return UINT64_MAX;
		if (filters[i].id != LZMA_FILTER_LZMA2) {
			if (filters[i].id < LZMA_FILTER_DELTA || filters[i].id > LZMA_FILTER_RISCV) return UINT64_MAX;
			continue;
		}
		if (filters[i].options == nullptr) return UINT64_MAX;
		const uint64_t d = ((const lzma_options_lzma *)filters[i].options)->dict_size;
		best = std::max<uint64_t>(best, d * 3 > (1u << 20) ? d * 3 : (1u << 20));
	}
	return best == 0 ? UINT64_MAX : best;
}

uint64_t lzma_stream_encoder_mt_memusage(const lzma_mt *options)
{
	xzb_lzma_options x; uint64_t bs;
	if (get_options(options, &x, &bs) != LZMA_OK) return UINT64_MAX;
	return WAVE_BLOCKS * bs * 112 + (1u << 20);  // device workspace per position, see DESIGN.md "HBM layout"
}

// stream_encoder_mt_update, common/stream_encoder_mt.c:914-950: a new filter chain for the Blocks that follow.  Allowed
// only between Blocks (the reference: no worker holds a partial Block); whole Blocks still waiting for their wave are
// encoded with the old options first.
static lzma_ret gpu_encoder_update(void *coder, const lzma_allocator *, const lzma_filter *filters, const lzma_filter *)
{
	GpuCoder *in = static_cast<GpuCoder *>(coder);
	if (in->kind != KIND_ENCODER || in->tail_done) return LZMA_PROG_ERROR;
	if (in->inbuf.size() % in->block_size != 0) return LZMA_PROG_ERROR;
	xzb_lzma_options x;
	std::vector<xzb_filter_spec> pre;
	if (parse_chain(filters, &x, &pre) != LZMA_OK || !valid_lzma2_options(x)) return LZMA_OPTIONS_ERROR;
	try {
		if (!in->inbuf.empty()) { const lzma_ret r = encode_prefix(in, in->inbuf.size()); if (r != LZMA_OK) return r; }
	} catch (const std::bad_alloc &) { return LZMA_MEM_ERROR; }
	for (xzb_ctx *c : in->pool) {
		const int rc = xzb_ctx_set_filters(c, pre.data(), (uint32_t)pre.size());
		if (rc != 0) return (lzma_ret)rc;
	}
	in->opt = x; in->pre = pre;
	return LZMA_OK;
}

// stream_decoder_memconfig, common/stream_decoder.c:389-408 (the figures are the reference's: what ITS decoder would allocate)
static lzma_ret gpu_decoder_memconfig(void *coder, uint64_t *memusage, uint64_t *old_memlimit, uint64_t new_memlimit)
{
	GpuCoder *in = static_cast<GpuCoder *>(coder);
	*memusage = in->memusage;
	*old_memlimit = in->memlimit;
	if (new_memlimit != 0) {
		if (new_memlimit < in->memusage) return LZMA_MEMLIMIT_ERROR;
		in->memlimit = new_memlimit;
	}
	return LZMA_OK;
}
static lzma_check gpu_decoder_get_check(const void *coder) { return (lzma_check)static_cast<const GpuCoder *>(coder)->cur_check; }

lzma_ret lzma_stream_encoder_mt(lzma_stream *strm, const lzma_mt *options)
{
	if (strm == nullptr) return LZMA_PROG_ERROR;
	xzb_lzma_options x; uint64_t bs = 0;
	std::vector<xzb_filter_spec> pre;
	const lzma_ret r0 = get_options(options, &x, &bs, &pre);
	if (r0 != LZMA_OK) return r0;
	if ((unsigned)options->check > 15) return LZMA_PROG_ERROR;       // stream_encoder_mt.c:1052-1056
	if (!lzma_check_is_supported(options->check)) return LZMA_UNSUPPORTED_CHECK;
	// option validation that the reference does in lzma_raw_encoder_memusage / filter init
	if (!valid_lzma2_options(x)) return LZMA_OPTIONS_ERROR;
	if (bs > (1ull << 30)) return LZMA_OPTIONS_ERROR;  // GPU path limit (DESIGN.md)
	const lzma_ret r = internal_create(strm, KIND_ENCODER, (uintptr_t)&lzma_stream_encoder_mt);
	if (r != LZMA_OK) return r;
	lzma_internal *si = strm->internal;
	GpuCoder *in = static_cast<GpuCoder *>(si->next.coder);
	in->opt = x; in->check = (uint32_t)options->check; in->block_size = bs;
	in->pre = pre;
	{
		// IDs, chain shape and Delta distances were checked above like lzma_raw_encoder_memusage does
		// (stream_encoder_mt.c:1073-1077).  What can still be wrong is a BCJ start offset that is not a multiple of the
		// filter's alignment: the reference finds that when a worker sets up its Block coder (simple_coder.c:276-278) and
		// reports LZMA_OPTIONS_ERROR from lzma_code, so it is kept for the first lzma_code call here too.
		const int rc = xzb_ctx_set_filters(in->ctx, in->pre.data(), (uint32_t)in->pre.size());
		if (rc != 0) { in->deferred = (lzma_ret)rc; in->pre.clear(); }
	}
	si->next.update = &gpu_encoder_update;
	si->supported_actions[LZMA_RUN] = true;  // stream_encoder_mt.c:1201-1205
	si->supported_actions[LZMA_FULL_FLUSH] = true;
	si->supported_actions[LZMA_FULL_BARRIER] = true;
	si->supported_actions[LZMA_FINISH] = true;
	return LZMA_OK;
}

static lzma_ret stream_decoder_create(lzma_stream *strm, uint64_t memlimit, uint32_t flags, uintptr_t marker)
{
	if (strm == nullptr) return LZMA_PROG_ERROR;
	if (flags & ~(LZMA_TELL_NO_CHECK | LZMA_TELL_UNSUPPORTED_CHECK | LZMA_TELL_ANY_CHECK | LZMA_CONCATENATED | LZMA_IGNORE_CHECK | LZMA_FAIL_FAST))
		return LZMA_OPTIONS_ERROR;  // stream_decoder.c:437-438
	const lzma_ret r = internal_create(strm, KIND_DECODER, marker);
	if (r != LZMA_OK) return r;
	lzma_internal *si = strm->internal;
	GpuCoder *in = static_cast<GpuCoder *>(si->next.coder);
	in->flags = flags;
	in->memlimit = memlimit > 1 ? memlimit : 1;  // stream_decoder.c:447: my_max(1, memlimit)
	si->next.get_check = &gpu_decoder_get_check;
	si->next.memconfig = &gpu_decoder_memconfig;
	si->supported_actions[LZMA_RUN] = true;
	si->supported_actions[LZMA_FINISH] = true;
	return LZMA_OK;
}

lzma_ret lzma_stream_decoder(lzma_stream *strm, uint64_t memlimit, uint32_t flags)
{
	return stream_decoder_create(strm, memlimit, flags, (uintptr_t)&lzma_stream_decoder);
}

lzma_ret lzma_stream_decoder_mt(lzma_stream *strm, const lzma_mt *options)
{
	if (strm == nullptr || options == nullptr) return LZMA_PROG_ERROR;
	if (options->threads == 0 || options->threads > 16384) return LZMA_OPTIONS_ERROR;  // stream_decoder_mt.c:1947-1949
	return stream_decoder_create(strm, options->memlimit_stop, options->flags, (uintptr_t)&lzma_stream_decoder_mt);
}

lzma_ret lzma_code(lzma_stream *strm, lzma_action action)  // common/common.c:203-376, generic over the coder vtable
{
	if (strm == nullptr || (strm->next_in == nullptr && strm->avail_in != 0) || (strm->next_out == nullptr && strm->avail_out != 0)
			|| strm->internal == nullptr || strm->internal->next.code == nullptr || (unsigned)action > 4
			|| !strm->internal->supported_actions[action])
		return LZMA_PROG_ERROR;
	if (strm->reserved_ptr1 != nullptr || strm->reserved_ptr2 != nullptr || strm->reserved_ptr3 != nullptr || strm->reserved_ptr4 != nullptr
			|| strm->reserved_int2 != 0 || strm->reserved_int3 != 0 || strm->reserved_int4 != 0
			|| strm->reserved_enum1 != LZMA_RESERVED_ENUM || strm->reserved_enum2 != LZMA_RESERVED_ENUM)
		return LZMA_OPTIONS_ERROR;
	lzma_internal *in = strm->internal;
	switch (in->sequence) {
	case ISEQ_RUN:
		switch (action) {
		case LZMA_RUN: break;
		case LZMA_SYNC_FLUSH: in->sequence = ISEQ_SYNC_FLUSH; break;
		case LZMA_FULL_FLUSH: in->sequence = ISEQ_FULL_FLUSH; break;
		case LZMA_FINISH: in->sequence = ISEQ_FINISH; break;
		case LZMA_FULL_BARRIER: in->sequence = ISEQ_FULL_BARRIER; break;
		}
		break;
	case ISEQ_SYNC_FLUSH: if (action != LZMA_SYNC_FLUSH || in->avail_in != strm->avail_in) return LZMA_PROG_ERROR; break;
	case ISEQ_FULL_FLUSH: if (action != LZMA_FULL_FLUSH || in->avail_in != strm->avail_in) return LZMA_PROG_ERROR; break;
	case ISEQ_FINISH: if (action != LZMA_FINISH || in->avail_in != strm->avail_in) return LZMA_PROG_ERROR; break;
	case ISEQ_FULL_BARRIER: if (action != LZMA_FULL_BARRIER || in->avail_in != strm->avail_in) return LZMA_PROG_ERROR; break;
	case ISEQ_END: return LZMA_STREAM_END;
	default: return LZMA_PROG_ERROR;
	}
	size_t in_pos = 0, out_pos = 0;
	lzma_ret ret = in->next.code(in->next.coder, strm->allocator, strm->next_in, &in_pos, strm->avail_in,
			strm->next_out, &out_pos, strm->avail_out, action);
	if (in_pos > 0) { strm->next_in += in_pos; strm->avail_in -= in_pos; strm->total_in += in_pos; }
	if (out_pos > 0) { strm->next_out += out_pos; strm->avail_out -= out_pos; strm->total_out += out_pos; }
	in->avail_in = strm->avail_in;
	switch (ret) {
	case LZMA_OK:
		if (out_pos == 0 && in_pos == 0) {
			if (in->allow_buf_error) ret = LZMA_BUF_ERROR; else in->allow_buf_error = true;
		} else {
			in->allow_buf_error = false;
		}
		break;
	case 101:  // LZMA_TIMED_OUT = LZMA_RET_INTERNAL1 (common.h:168): a coder's timeout is LZMA_OK without the LZMA_BUF_ERROR bookkeeping
		in->allow_buf_error = false;
		ret = LZMA_OK;
		break;
	case LZMA_SEEK_NEEDED:
		in->allow_buf_error = false;
		if (in->sequence == ISEQ_FINISH) in->sequence = ISEQ_RUN;
		break;
	case LZMA_STREAM_END:
		if (in->sequence == ISEQ_SYNC_FLUSH || in->sequence == ISEQ_FULL_FLUSH || in->sequence == ISEQ_FULL_BARRIER) in->sequence = ISEQ_RUN;
		else in->sequence = ISEQ_END;
		in->allow_buf_error = false;
		break;
	case LZMA_NO_CHECK: case LZMA_UNSUPPORTED_CHECK: case LZMA_GET_CHECK: case LZMA_MEMLIMIT_ERROR:
		in->allow_buf_error = false;
		break;
	default:
		in->sequence = ISEQ_ERROR;
		break;
	}
	return ret;
}

// common/common.c:436-476: through the coder's memconfig; coders without one (the encoders) report 0 / LZMA_PROG_ERROR
uint64_t lzma_memusage(const lzma_stream *strm)
{
	uint64_t memusage, old_memlimit;
	if (strm == nullptr || strm->internal == nullptr || strm->internal->next.memconfig == nullptr
			|| strm->internal->next.memconfig(strm->internal->next.coder, &memusage, &old_memlimit, 0) != LZMA_OK)
		return 0;
	return memusage;
}
uint64_t lzma_memlimit_get(const lzma_stream *strm)
{
	uint64_t memusage, old_memlimit;
	if (strm == nullptr || strm->internal == nullptr || strm->internal->next.memconfig == nullptr
			|| strm->internal->next.memconfig(strm->internal->next.coder, &memusage, &old_memlimit, 0) != LZMA_OK)
		return 0;
	return old_memlimit;
}
lzma_ret lzma_memlimit_set(lzma_stream *strm, uint64_t new_memlimit)
{
	uint64_t memusage, old_memlimit;
	if (strm == nullptr || strm->internal == nullptr || strm->internal->next.memconfig == nullptr) return LZMA_PROG_ERROR;
	if (new_memlimit == 0) new_memlimit = 1;
	return strm->internal->next.memconfig(strm->internal->next.coder, &memusage, &old_memlimit, new_memlimit);
}

lzma_check lzma_get_check(const lzma_stream *strm)  // common/common.c:422-433
{
	if (strm == nullptr || strm->internal == nullptr || strm->internal->next.get_check == nullptr) return LZMA_CHECK_NONE;
	return strm->internal->next.get_check(strm->internal->next.coder);
}

void lzma_end(lzma_stream *strm)  // common/common.c:379-389
{
	if (strm != nullptr && strm->internal != nullptr) internal_destroy(strm);
}

void lzma_get_progress(lzma_stream *strm, uint64_t *progress_in, uint64_t *progress_out)  // common/common.c:406-419
{
	if (strm->internal != nullptr && strm->internal->next.get_progress != nullptr)
		strm->internal->next.get_progress(strm->internal->next.coder, progress_in, progress_out);
	else { *progress_in = strm->total_in; *progress_out = strm->total_out; }
}

// lzma_filters_update, common/filter_encoder.c:210-241: validate, reverse, hand to the coder's `update`.  In the hybrid
// the reference's own validator is used when it is loaded (any chain it accepts may go to ITS coders); the GPU encoder's
// update accepts LZMA2-only chains.
extern uint64_t lzma_raw_encoder_memusage(const lzma_filter *filters) __attribute__((weak));
lzma_ret lzma_filters_update(lzma_stream *strm, const lzma_filter *filters)
{
	if (strm == nullptr || strm->internal == nullptr || strm->internal->next.update == nullptr) return LZMA_PROG_ERROR;
	if (filters == nullptr) return LZMA_PROG_ERROR;
	if (&lzma_raw_encoder_memusage != nullptr && lzma_raw_encoder_memusage(filters) == UINT64_MAX) return LZMA_OPTIONS_ERROR;
	size_t count = 1;
	while (filters[count].id != LZMA_VLI_UNKNOWN) { if (++count > 4) return LZMA_OPTIONS_ERROR; }
	lzma_filter reversed_filters[5];
	for (size_t i = 0; i < count; ++i) reversed_filters[count - i - 1] = filters[i];
	reversed_filters[count].id = LZMA_VLI_UNKNOWN;
	return strm->internal->next.update(strm->internal->next.coder, strm->allocator, filters, reversed_filters);
}

}  // extern "C"
