// xzb_frame.cuh -- the .xz container: framing around the LZMA2 payload of one block, plus the
// Stream Header / Index / Stream Footer, written (host/device) and read back (host only, at the end).
// Reference: common/block_header_encoder.c, common/block_encoder.c:104-133,
// common/block_buffer_encoder.c:27-162, common/vli_encoder.c, common/index_encoder.c:43-165,
// common/stream_flags_encoder.c:29-85; the read side: common/vli_decoder.c,
// common/block_header_decoder.c, common/index_hash.c, common/stream_flags_decoder.c.
#pragma once
#include "xzb_common.cuh"
#include "xzb_filters.cuh"
#include "../../include/xzb200.h"

XZB_HD uint32_t xzb_vli_put(uint8_t *out, uint64_t v)  // vli_encoder.c:16-69 (single call)
{
	uint32_t n = 0;
	while (v >= 0x80) { out[n++] = (uint8_t)v | 0x80; v >>= 7; }
	out[n++] = (uint8_t)v;
	return n;
}
XZB_HD uint32_t xzb_vli_size(uint64_t v) { uint32_t n = 0; do { v >>= 7; ++n; } while (v != 0); return n; }  // vli_size.c:15-30

XZB_HD uint32_t xzb_crc32_bytes(const uint32_t *table, const uint8_t *buf, uint32_t size, uint32_t crc)
{
	crc = ~crc;
	for (uint32_t i = 0; i < size; ++i) crc = table[(crc ^ buf[i]) & 0xFF] ^ (crc >> 8);
	return ~crc;
}

XZB_HD uint32_t xzb_check_size(uint32_t check) { return check == 0 ? 0 : check == 1 ? 4 : check == 4 ? 8 : check == 10 ? 32 : 0xFFFFFFFFu; }  // CRC32, CRC64, SHA-256

// lzma2_bound + lzma_block_buffer_bound64, block_buffer_encoder.c:27-71
XZB_HD uint64_t xzb_lzma2_bound(uint64_t u) { return u + ((u + XZB_LZMA2_CHUNK_MAX - 1) / XZB_LZMA2_CHUNK_MAX) * 3 + 1; }
XZB_HD uint64_t xzbi_block_bound(uint64_t u) { return 92 + ((xzb_lzma2_bound(u) + 3) & ~(uint64_t)3); }

// lzma_block_header_size :16-68 with both sizes present: LZMA2 last, ff_len bytes of Filter Flags of the filters before it
XZB_HD uint32_t xzb_block_header_size(uint64_t comp, uint64_t uncomp, uint32_t ff_len = 0) { return (6 + xzb_vli_size(comp) + xzb_vli_size(uncomp) + ff_len + 3 + 3) & ~3u; }

// lzma_block_header_encode :71-131
XZB_HD void xzb_block_header_encode(const uint32_t *crc32_table, uint8_t *out, uint32_t header_size, uint64_t comp, uint64_t uncomp, uint8_t dict_prop,
		const uint8_t *ff = nullptr, uint32_t ff_len = 0, uint32_t n_pre = 0)
{
	const uint32_t out_size = header_size - 4;
	out[0] = (uint8_t)(out_size / 4);
	out[1] = (uint8_t)(0xC0 | n_pre);   // both sizes present, number of filters - 1
	uint32_t pos = 2;
	pos += xzb_vli_put(out + pos, comp);
	pos += xzb_vli_put(out + pos, uncomp);
	for (uint32_t i = 0; i < ff_len; ++i) out[pos++] = ff[i];   // filter_flags_encoder.c:31-56 for the Delta / BCJ filters
	out[pos++] = 0x21; out[pos++] = 0x01; out[pos++] = dict_prop;  // filter_flags_encoder.c:31-56
	while (pos < out_size) out[pos++] = 0;
	const uint32_t crc = xzb_crc32_bytes(crc32_table, out, out_size, 0);
	for (int i = 0; i < 4; ++i) out[out_size + i] = (uint8_t)(crc >> (8 * i));
}

// lzma_lzma2_props_encode, lzma/lzma2_encoder.c:375-400
XZB_HD uint8_t xzb_lzma2_dict_prop(uint32_t dict_size)
{
	uint32_t d = dict_size > 4096 ? dict_size : 4096;
	--d; d |= d >> 2; d |= d >> 3; d |= d >> 4; d |= d >> 8; d |= d >> 16;
	if (d == 0xFFFFFFFFu) return 40;
	return (uint8_t)(xzb_dist_slot(d + 1) - 24);
}

XZB_HD uint32_t xzb_stream_header(const uint32_t *crc32_table, uint8_t *out, uint32_t check)  // stream_flags_encoder.c:29-53
{
	out[0] = 0xFD; out[1] = 0x37; out[2] = 0x7A; out[3] = 0x58; out[4] = 0x5A; out[5] = 0x00;
	out[6] = 0x00; out[7] = (uint8_t)check;
	const uint32_t crc = xzb_crc32_bytes(crc32_table, out + 6, 2, 0);
	for (int i = 0; i < 4; ++i) out[8 + i] = (uint8_t)(crc >> (8 * i));
	return 12;
}
XZB_HD uint32_t xzb_stream_footer(const uint32_t *crc32_table, uint8_t *out, uint32_t check, uint64_t index_size)  // :56-85
{
	const uint32_t bs = (uint32_t)(index_size / 4 - 1);
	for (int i = 0; i < 4; ++i) out[4 + i] = (uint8_t)(bs >> (8 * i));
	out[8] = 0x00; out[9] = (uint8_t)check;
	const uint32_t crc = xzb_crc32_bytes(crc32_table, out + 4, 6, 0);
	for (int i = 0; i < 4; ++i) out[i] = (uint8_t)(crc >> (8 * i));
	out[10] = 'Y'; out[11] = 'Z';
	return 12;
}
// index_encode, index_encoder.c:43-165; out == NULL returns the size only
XZB_HD uint64_t xzbi_index_encode(const uint32_t *crc32_table, const uint64_t *unpadded, const uint64_t *uncompressed, uint64_t count, uint8_t *out)
{
	uint64_t n = 1 + xzb_vli_size(count);
	for (uint64_t i = 0; i < count; ++i) n += xzb_vli_size(unpadded[i]) + xzb_vli_size(uncompressed[i]);
	const uint64_t padded = (n + 3) & ~(uint64_t)3;
	if (out == 0) return padded + 4;
	uint64_t pos = 0;
	out[pos++] = 0x00;
	pos += xzb_vli_put(out + pos, count);
	for (uint64_t i = 0; i < count; ++i) { pos += xzb_vli_put(out + pos, unpadded[i]); pos += xzb_vli_put(out + pos, uncompressed[i]); }
	while (pos < padded) out[pos++] = 0x00;
	uint32_t crc = 0xFFFFFFFFu;  // incremental form of xzb_crc32_bytes for 64-bit sizes
	for (uint64_t i = 0; i < pos; ++i) crc = crc32_table[(crc ^ out[i]) & 0xFF] ^ (crc >> 8);
	crc = ~crc;
	for (int i = 0; i < 4; ++i) out[pos++] = (uint8_t)(crc >> (8 * i));
	return pos;
}

// ---- per-block framing as worker_encode() does it (common/stream_encoder_mt.c:218-359) ----
struct XzbBlockResult {
	uint32_t total_size;     // bytes of the finished Block (header + data + padding + check)
	uint32_t header_size;
	uint64_t unpadded_size;  // lzma_block_unpadded_size(), block_util.c:53-77
	uint32_t fallback;       // 1 = stored with uncompressed LZMA2 chunks (block_buffer_encoder.c:87-162)
	uint32_t ret;            // XZB_OK or error
	uint32_t n_symbols, n_chunks_lzma, n_chunks_raw, pad_;
};

// `bytes` = the Check field as stored: little-endian CRC (check.c:146-165) or the 32 SHA-256 bytes
XZB_HD void xzb_put_check(uint8_t *out, uint32_t check, const uint8_t *bytes)
{
	const uint32_t n = xzb_check_size(check);
	for (uint32_t i = 0; i < n; ++i) out[i] = bytes[i];
}

// Normal path: payload already sits at out[header_size .. payload_end).  Returns false when the
// block does not fit -> caller takes the raw fallback.  Two framings:
//  oneshot == 0  worker_encode(): header + data + padding + check must fit
//                out_size = lzma_block_buffer_bound64(block_size) (stream_encoder_mt.c:225-344);
//  oneshot == 1  lzma_block_buffer_encode(): the LZMA2 data alone must fit
//                out_size = header_size + lzma2_bound(in_size) (block_buffer_encoder.c:165-210).
XZB_HD bool xzb_block_finish_normal(const uint32_t *crc32_table, uint8_t *out, uint32_t payload_end, uint32_t header_size,
		uint64_t out_size, uint32_t oneshot, uint32_t check, const uint8_t *check_bytes, uint32_t in_size, uint8_t dict_prop, XzbBlockResult *res,
		const uint8_t *ff = nullptr, uint32_t ff_len = 0, uint32_t n_pre = 0)
{
	const uint32_t csize = xzb_check_size(check);
	const uint32_t comp = payload_end - header_size;
	const uint32_t pad = (4 - (comp & 3)) & 3;
	if ((uint64_t)payload_end + (oneshot ? 0 : pad + csize) > out_size) return false;
	uint32_t pos = payload_end;
	for (uint32_t i = 0; i < pad; ++i) out[pos++] = 0;  // block_encoder.c:104-112
	xzb_put_check(out + pos, check, check_bytes);
	pos += csize;
	xzb_block_header_encode(crc32_table, out, header_size, comp, in_size, dict_prop, ff, ff_len, n_pre);
	res->total_size = pos; res->header_size = header_size;
	res->unpadded_size = (uint64_t)header_size + comp + csize;
	res->fallback = 0;
	return true;
}

// Raw fallback (the UNFILTERED input under an LZMA2-only header, block_buffer_encoder.c:87-162), work-shared by `nthreads` workers (tid in [0, nthreads)); worker 0 also writes
// header, control bytes, end marker, padding and check.  lzma_block_uncomp_encode.
XZB_HD void xzb_block_finish_raw(const uint32_t *crc32_table, const uint8_t *in, uint32_t in_size, uint8_t *out,
		uint32_t check, const uint8_t *check_bytes, XzbBlockResult *res, uint32_t tid, uint32_t nthreads)
{
	const uint64_t comp = xzb_lzma2_bound(in_size);
	const uint32_t hs = xzb_block_header_size(comp, in_size);
	const uint32_t csize = xzb_check_size(check);
	// payload copy: chunk c covers in[c*65536 ..), lands at hs + c*(65536+3) + 3
	for (uint32_t i = tid; i < in_size; i += nthreads) {
		const uint32_t c = i >> 16;
		out[hs + c * 3 + 3 + i] = in[i];
	}
	if (tid == 0) {
		xzb_block_header_encode(crc32_table, out, hs, comp, in_size, 0x00);
		const uint32_t nchunks = (in_size + XZB_LZMA2_CHUNK_MAX - 1) / XZB_LZMA2_CHUNK_MAX;
		for (uint32_t c = 0; c < nchunks; ++c) {
			const uint32_t off = c * XZB_LZMA2_CHUNK_MAX;
			const uint32_t copy = in_size - off < XZB_LZMA2_CHUNK_MAX ? in_size - off : XZB_LZMA2_CHUNK_MAX;
			uint8_t *h = out + hs + c * 3 + off;
			h[0] = c == 0 ? 0x01 : 0x02;
			h[1] = (uint8_t)((copy - 1) >> 8); h[2] = (uint8_t)((copy - 1) & 0xFF);
		}
		uint32_t pos = hs + nchunks * 3 + in_size;
		out[pos++] = 0x00;
		for (uint64_t i = comp; i & 3; ++i) out[pos++] = 0x00;
		xzb_put_check(out + pos, check, check_bytes);
		pos += csize;
		res->total_size = pos; res->header_size = hs;
		res->unpadded_size = (uint64_t)hs + comp + csize;
		res->fallback = 1;
	}
}

// ---- read side (host only), over untrusted input: every reader stays inside the `size` / `avail` bytes it is given ----
static inline uint32_t xzb_check_field_size(uint32_t check)  // any of the 16 Check IDs, supported or not (check.c:62-86)
{
	static const uint8_t sizes[16] = { 0, 4, 4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64 };
	return check > 15 ? 0xFFFFFFFFu : sizes[check];
}

static inline uint32_t xzb_rd32(const uint8_t *p) { return p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// lzma_vli_decode (single call), vli_decoder.c:16-86.  Whatever the result, *v has the bits read so far and *pos is past
// the last byte read, so that a lax reader can still use what a strict one rejects.  LONG and NONMIN are invalid.
enum { XZB_VLI_OK, XZB_VLI_SHORT /* input ran out */, XZB_VLI_LONG /* no last byte in nine */, XZB_VLI_NONMIN /* last byte 0x00 */ };
static inline int xzb_vli_get(const uint8_t *in, uint64_t *pos, uint64_t size, uint64_t *v)
{
	*v = 0;
	for (uint32_t i = 0; i < 9; ++i) {
		if (*pos >= size) return XZB_VLI_SHORT;
		const uint8_t b = in[(*pos)++];
		*v |= (uint64_t)(b & 0x7F) << (7 * i);
		if ((b & 0x80) == 0) return (b == 0x00 && i != 0) ? XZB_VLI_NONMIN : XZB_VLI_OK;
	}
	return XZB_VLI_LONG;
}
static inline int xzb_vli_verdict(int st) { return st == XZB_VLI_OK ? XZB_OK : st == XZB_VLI_SHORT ? XZB_BUF_ERROR : XZB_DATA_ERROR; }

// Stream Header / Footer, stream_flags_decoder.c:26-83, with the verdicts in the reference's order.  Comparing the
// footer's Index size and Check ID with the Index and the Stream Header is the caller's.
static inline int xzb_stream_header_decode(const uint32_t *crc32_table, const uint8_t in[12], uint32_t *check)
{
	static const uint8_t magic[6] = { 0xFD, 0x37, 0x7A, 0x58, 0x5A, 0x00 };
	for (int i = 0; i < 6; ++i) if (in[i] != magic[i]) return XZB_FORMAT_ERROR;
	if (xzb_crc32_bytes(crc32_table, in + 6, 2, 0) != xzb_rd32(in + 8)) return XZB_DATA_ERROR;
	if (in[6] != 0x00 || (in[7] & 0xF0)) return XZB_OPTIONS_ERROR;
	*check = in[7] & 0x0F;
	return XZB_OK;
}
static inline int xzb_stream_footer_decode(const uint32_t *crc32_table, const uint8_t in[12], uint32_t *check, uint64_t *index_size)
{
	if (in[10] != 'Y' || in[11] != 'Z' || xzb_crc32_bytes(crc32_table, in + 4, 6, 0) != xzb_rd32(in)) return XZB_DATA_ERROR;
	if (in[8] != 0x00 || (in[9] & 0xF0)) return XZB_OPTIONS_ERROR;
	*check = in[9] & 0x0F;
	*index_size = ((uint64_t)xzb_rd32(in + 4) + 1) * 4;  // Backward Size
	return XZB_OK;
}

// Block Header framing only (block_header_decoder.c:17-73): Header Size, flags, and the sizes the flags announce, read
// inside the whole header (CRC32 included), each with its bits so far, its end offset and its xzb_vli_get result; an
// absent one is 0, zero bytes long, OK.  No CRC32 or filter checks.  False when the header is not all in `avail`.
struct XzbVliField { uint64_t v; uint32_t end; int st; };
struct XzbBlockFraming { uint32_t hsize; uint8_t flags; XzbVliField comp, uncomp; };
static inline bool xzb_block_framing(const uint8_t *h, uint64_t avail, XzbBlockFraming *f)
{
	f->hsize = ((uint32_t)h[0] + 1) * 4;
	if (avail < f->hsize) return false;
	f->flags = h[1];
	uint64_t pos = 2;
	f->comp = XzbVliField{ 0, 2, XZB_VLI_OK };
	if (f->flags & 0x40) { f->comp.st = xzb_vli_get(h, &pos, f->hsize, &f->comp.v); f->comp.end = (uint32_t)pos; }
	f->uncomp = XzbVliField{ 0, (uint32_t)pos, XZB_VLI_OK };
	if (f->flags & 0x80) { f->uncomp.st = xzb_vli_get(h, &pos, f->hsize, &f->uncomp.v); f->uncomp.end = (uint32_t)pos; }
	return true;
}

// The full Block Header parse, block_header_decoder.c:17-124 (XZB_BUF_ERROR: not all in `avail`): LZMA2 last, up to
// three Delta / BCJ filters in front of it.
struct XzbBlockHeader {
	uint64_t hsize, comp, uncomp;  // comp/uncomp = UINT64_MAX when absent
	uint32_t dict_size;
	uint32_t n_pre;                // filters in front of LZMA2, in chain (= encoding) order
	XzbPreFilter pre[3];
};
static inline int xzb_block_header_decode(const uint32_t *crc32_table, const uint8_t *h, uint64_t avail, XzbBlockHeader *hb)
{
	XzbBlockFraming f;
	if (!xzb_block_framing(h, avail, &f)) return XZB_BUF_ERROR;
	const uint64_t hin = f.hsize - 4;
	if (xzb_crc32_bytes(crc32_table, h, (uint32_t)hin, 0) != xzb_rd32(h + hin)) return XZB_DATA_ERROR;
	if (f.flags & 0x3C) return XZB_OPTIONS_ERROR;
	if (f.comp.st != XZB_VLI_OK || f.uncomp.st != XZB_VLI_OK || f.uncomp.end > hin) return XZB_DATA_ERROR;  // uncomp.end >= comp.end
	hb->comp = (f.flags & 0x40) ? f.comp.v : UINT64_MAX;
	hb->uncomp = (f.flags & 0x80) ? f.uncomp.v : UINT64_MAX;
	if (hb->comp == 0 || (hb->comp != UINT64_MAX && hb->comp > (UINT64_MAX / 2 - 1024 - 64 - 4))) return XZB_DATA_ERROR;
	uint64_t hp = f.uncomp.end;
	const uint32_t nfilters = (f.flags & 3) + 1;
	bool have = false;
	hb->n_pre = 0;
	for (uint32_t i = 0; i < nfilters; ++i) {  // lzma_filter_flags_decode, filter_flags_decoder.c:16-45
		uint64_t id, psize;
		if (xzb_vli_get(h, &hp, hin, &id) != XZB_VLI_OK || id >= (1ull << 62)) return XZB_DATA_ERROR;
		if (xzb_vli_get(h, &hp, hin, &psize) != XZB_VLI_OK || hin - hp < psize) return XZB_DATA_ERROR;
		if (i + 1 < nfilters) {
			// a filter in front of the last one: Delta or BCJ (LZMA2 may only be last, validate_chain, filter_common.c:122-249)
			if (id > 0xFF || !xzb_filter_known((uint32_t)id)) return XZB_OPTIONS_ERROR;
			XzbPreFilter &pf = hb->pre[hb->n_pre++];
			pf.id = (uint32_t)id; pf.arg = 0;
			if (id == XZB_FILTER_DELTA) {          // lzma_delta_props_decode, delta_decoder.c:66-87
				if (psize != 1) return XZB_OPTIONS_ERROR;
				pf.arg = (uint32_t)h[hp] + 1;
			} else {                               // lzma_simple_props_decode, simple_decoder.c:15-39
				if (psize == 4) pf.arg = xzb_rd32(h + hp);
				else if (psize != 0) return XZB_OPTIONS_ERROR;
				if (pf.arg & (xzb_filter_alignment(pf.id) - 1)) return XZB_OPTIONS_ERROR;
			}
			hp += psize;
			continue;
		}
		if (id != XZB_FILTER_LZMA2) return XZB_OPTIONS_ERROR;
		if (psize != 1 || (h[hp] & 0xC0) || h[hp] > 40) return XZB_OPTIONS_ERROR;  // lzma_lzma2_props_decode, lzma2_decoder.c:298-331
		hb->dict_size = h[hp] == 40 ? 0xFFFFFFFFu : (2u | (h[hp] & 1u)) << (h[hp] / 2u + 11);
		hp += psize; have = true;
	}
	while (hp < hin) if (h[hp++] != 0x00) return XZB_OPTIONS_ERROR;
	if (!have) return XZB_OPTIONS_ERROR;
	hb->hsize = f.hsize;
	return XZB_OK;
}

// Index, index_hash.c:175-341, from its Indicator at in[0].  The records are walked to their end whatever their VLIs
// hold, so that a lax reader learns where the Index ends; the verdict is the first fault in stream order, a count or
// record that differs from *want (when given) included.
struct XzbIndexWant { const xzb_index_record *recs; uint64_t n; };
struct XzbIndexRead {
	uint64_t count;  // Number of Records as stored
	bool listed;     // false: the input ran out within the records
	uint64_t end;    // when listed: just past the CRC32 (the records rounded up to four bytes, + 4)
	uint64_t stop;   // where a strict reader stops: just past the first fault, else = end
};
static inline int xzb_index_read(const uint32_t *crc32_table, const uint8_t *in, uint64_t size, const XzbIndexWant *want, XzbIndexRead *x)
{
	uint64_t pos = 1, u = 0, w = 0;
	int ret = XZB_OK, st;
	auto fault = [&](int verdict) { if (ret == XZB_OK && verdict != XZB_OK) { ret = verdict; x->stop = pos; } };
	fault(xzb_vli_verdict(st = xzb_vli_get(in, &pos, size, &x->count)));
	if (want != nullptr && x->count != want->n) fault(XZB_DATA_ERROR);
	for (uint64_t r = 0; st != XZB_VLI_SHORT && r < x->count; ++r) {
		fault(xzb_vli_verdict(st = xzb_vli_get(in, &pos, size, &u)));
		if (st != XZB_VLI_SHORT) fault(xzb_vli_verdict(st = xzb_vli_get(in, &pos, size, &w)));
		if (ret == XZB_OK && want != nullptr && (u != want->recs[r].unpadded_size || w != want->recs[r].uncompressed_size)) fault(XZB_DATA_ERROR);
	}
	x->listed = st != XZB_VLI_SHORT;
	x->end = ((pos + 3) & ~(uint64_t)3) + 4;
	while (ret == XZB_OK && (pos & 3)) fault(pos >= size ? XZB_BUF_ERROR : in[pos++] != 0x00 ? XZB_DATA_ERROR : XZB_OK);
	if (size - pos < 4) fault(XZB_BUF_ERROR);
	if (ret != XZB_OK) return ret;
	uint32_t crc = 0xFFFFFFFFu;  // xzb_crc32_bytes for a 64-bit length
	for (uint64_t i = 0; i < pos; ++i) crc = crc32_table[(crc ^ in[i]) & 0xFF] ^ (crc >> 8);
	x->stop = pos + 4;
	return ~crc != xzb_rd32(in + pos) ? XZB_DATA_ERROR : XZB_OK;
}
