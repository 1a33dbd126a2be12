// xzb_dec_stream.cuh -- the Stream decoder's walk over one .xz Stream, as step functions that the host driver
// (decode_streams) and the device driver (xzb_k_dec_scan / xzb_k_dec_settle) both run (host and device).
// Reference: common/stream_decoder.c:101-378, block_decoder.c:64-200, index_hash.c:175-341, and for the runs of sized
// Blocks decoded side by side stream_decoder_mt.c:862-931.
//
// One round of a Stream:
//   xzb_dec_scan    the Stream Header (first round), then the next run of Blocks: Blocks whose headers carry both sizes
//                   run together, an unsized Block runs alone; each gets the input and output room its decode job may use;
//   (the caller decodes the run's Blocks, undoes their Delta / BCJ filters and computes their integrity checks)
//   xzb_dec_settle  validates the run's results in Stream order: decoder verdicts, sizes, padding, Check field; appends
//                   an Index record per good Block; runs xzb_dec_end when the Stream failed or reached its Index;
//   xzb_dec_end     the Index against the records, then the Stream Footer.
#pragma once
#include "xzb_common.cuh"
#include "xzb_dec.cuh"
#include "xzb_frame.cuh"

struct XzbDecResult { uint32_t ret, in_used, out_used, pad_; };  // what xzb_lzma2_decode returned for one Block

// The cursor over one Stream: a plain struct, so that it can live in device memory.
struct XzbDecCursor {
	uint64_t in_size, out_cap;
	uint32_t flags;
	// results
	int32_t ret;
	int32_t buf_reason;       // why XZB_BUF_ERROR: 1 = the input ended early, 2 = the output is too small
	uint32_t done;
	uint64_t in_used, out_size;
	// cursor
	uint32_t at_index, check, csize, verify;
	uint64_t ip, op;          // ip == 0: the Stream Header is not read yet
	uint64_t n_recs;          // Index records so far (the caller's array)
	uint64_t bip;             // where the current run's scan stopped
	int32_t pending;          // error found while scanning ahead: reported after the round
	uint32_t nb;              // Blocks in the current run
};

// One Block of a run as xzb_dec_scan found it: its header, where it sits, and the room its decode job gets.
struct XzbDecBlk {
	XzbBlockHeader hb;
	uint64_t hdr_off, out_off;   // in the Stream's input / output
	uint32_t in_avail, out_limit;
	uint32_t truncated;          // the input ends inside the Compressed Data: running out of it is XZB_BUF_ERROR
	uint32_t out_exact;          // out_limit is the Uncompressed Size: wanting more is XZB_DATA_ERROR
};

XZB_HD void xzb_dec_init(XzbDecCursor &s, uint64_t in_size, uint64_t out_cap, uint32_t flags, uint64_t n_prior)
{
	s.in_size = in_size; s.out_cap = out_cap; s.flags = flags;
	s.ret = XZB_OK; s.buf_reason = 1; s.done = 0; s.in_used = 0; s.out_size = 0;
	s.at_index = 0; s.check = 0; s.csize = 0; s.verify = 1;
	s.ip = 0; s.op = 0; s.n_recs = n_prior; s.bip = 0; s.pending = XZB_OK; s.nb = 0;
}

// Index + Stream Footer behind the last Block (common/index_hash.c:175-341, stream_decoder.c:266-332), then the
// Stream's results.  recs[0 .. s.n_recs) are the Blocks' Index records.
XZB_HD void xzb_dec_end(XzbDecCursor &s, const uint8_t *in, const uint32_t *crc32_table, const xzb_index_record *recs)
{
	if (s.ret == XZB_OK) {
		const XzbIndexWant want{ recs, s.n_recs };
		XzbIndexRead x;
		s.ret = xzb_index_read(crc32_table, in + s.ip, s.in_size - s.ip, &want, &x);
		s.ip += x.stop;
		uint32_t fcheck = 0; uint64_t fisize = 0;
		if (s.ret == XZB_OK && s.in_size - s.ip < 12) s.ret = XZB_BUF_ERROR;
		if (s.ret == XZB_OK) s.ret = xzb_stream_footer_decode(crc32_table, in + s.ip, &fcheck, &fisize);
		if (s.ret == XZB_OK && (fisize != x.end || fcheck != s.check)) s.ret = XZB_DATA_ERROR;
		if (s.ret == XZB_OK) s.ip += 12;
	}
	s.in_used = s.ip;
	s.out_size = s.op;
	s.done = 1;
}

// The Stream Header; false when the Stream is already finished by it.
XZB_HD bool xzb_dec_header(XzbDecCursor &s, const uint8_t *in, const uint32_t *crc32_table)
{
	if (s.ip != 0) return !s.done;
	const int hr = s.in_size < 12 ? XZB_BUF_ERROR : xzb_stream_header_decode(crc32_table, in, &s.check);
	if (hr != XZB_OK) { s.ret = hr; s.done = 1; return false; }
	s.csize = xzb_check_field_size(s.check);
	// Checks other than CRC32 / CRC64 / SHA-256 are reserved IDs: like the reference
	// (block_decoder.c:178-190 compares only when lzma_check_is_supported()) they are skipped.
	s.verify = !(s.flags & XZB_DEC_IGNORE_CHECK);  // LZMA_IGNORE_CHECK, stream_decoder.c:188-190
	s.ip = 12;
	return true;
}

// The Check ID whose value the caller computes for each Block of this Stream's runs: 1, 4, 10, or 0 for none.
XZB_HD uint32_t xzb_dec_check_computed(const XzbDecCursor &s) { return s.verify && (s.check == 1 || s.check == 4 || s.check == 10) ? s.check : 0; }

// Scans the next run of at most `max` Blocks (max > 0) and returns how many it holds; blks (when given) receives them.
// A run of none ends the Stream (xzb_dec_end).  The cursor keeps the run for xzb_dec_settle.
XZB_HD uint32_t xzb_dec_scan(XzbDecCursor &s, const uint8_t *in, const uint32_t *crc32_table, XzbDecBlk *blks, uint32_t max,
		const xzb_index_record *recs)
{
	s.nb = 0;
	if (!xzb_dec_header(s, in, crc32_table)) return 0;
	// gather a run of blocks whose headers carry both sizes (stream_decoder_mt.c:862-931)
	s.pending = XZB_OK;
	s.bip = s.ip;
	uint64_t bop = s.op;
	uint32_t nb = 0;
	for (;;) {
		if (s.bip >= s.in_size) { s.pending = XZB_BUF_ERROR; break; }
		if (in[s.bip] == 0x00) { s.at_index = 1; break; }
		XzbBlockHeader hb;
		const int r = xzb_block_header_decode(crc32_table, in + s.bip, s.in_size - s.bip, &hb);
		if (r != XZB_OK) { s.pending = r; break; }
		const bool sized = hb.comp != UINT64_MAX && hb.uncomp != UINT64_MAX;
		if (!sized && nb != 0) break;  // decode what we have first
		if (blks != nullptr) {
			XzbDecBlk &k = blks[nb];
			k.hb = hb; k.hdr_off = s.bip; k.out_off = bop;
			k.truncated = 1; k.out_exact = 0;
			const uint64_t dpos = s.bip + hb.hsize;
			uint64_t in_avail = s.in_size - dpos;
			if (hb.comp != UINT64_MAX && hb.comp <= in_avail) { in_avail = hb.comp; k.truncated = 0; }
			uint64_t out_limit = s.out_cap - bop;
			if (hb.uncomp != UINT64_MAX && hb.uncomp <= out_limit) { out_limit = hb.uncomp; k.out_exact = 1; }
			k.in_avail = (uint32_t)(in_avail < 0xFFFFFFF0ull ? in_avail : 0xFFFFFFF0ull);
			k.out_limit = (uint32_t)(out_limit < 0xFFFFFFF0ull ? out_limit : 0xFFFFFFF0ull);
		}
		++nb;
		if (!sized) break;  // direct mode: one block at a time
		const uint64_t padded = (hb.comp + 3) & ~3ull;
		if (s.in_size - (s.bip + hb.hsize) < padded + s.csize || s.out_cap - bop < hb.uncomp) break;  // let the per-block logic report it
		s.bip += hb.hsize + padded + s.csize; bop += hb.uncomp;
		if (nb >= max) break;
	}
	if (nb == 0) { s.ret = s.pending; xzb_dec_end(s, in, crc32_table, recs); return 0; }
	s.nb = nb;
	return nb;
}

// Validates the current run in Stream order (common/block_decoder.c:64-200).  Block b of the run has its header in
// blks[b], its decode result in res[b] and, when xzb_dec_check_computed(s) != 0, the computed check at
// chk + b * chk_stride in the Check field's byte order.  Like the reference (lz_decoder.c:128-160 copies what was
// decoded before it looks at the return code), the bytes a failing Block produced before the error are still
// delivered.  Appends the good Blocks' Index records to recs (room for rec_cap) and returns the bytes they produced.
XZB_HD uint64_t xzb_dec_settle(XzbDecCursor &s, const uint8_t *in, const uint32_t *crc32_table, const XzbDecBlk *blks,
		const XzbDecResult *res, const uint8_t *chk, uint32_t chk_stride, xzb_index_record *recs, uint64_t rec_cap)
{
	uint64_t produced = 0;
	const bool cmp = xzb_dec_check_computed(s) != 0;
	for (uint32_t b = 0; b < s.nb && s.ret == XZB_OK; ++b) {
		const XzbBlockHeader &hb = blks[b].hb;
		const XzbDecResult &r = res[b];
		const uint64_t op_fail = blks[b].out_off + r.out_used;
		int ret = XZB_OK;
		if (r.ret == XZB_NEED_INPUT) ret = blks[b].truncated ? XZB_BUF_ERROR : XZB_DATA_ERROR;
		else if (r.ret == XZB_NEED_OUTPUT) { ret = blks[b].out_exact ? XZB_DATA_ERROR : XZB_BUF_ERROR; s.buf_reason = 2; }
		else if (r.ret != XZB_OK) ret = (int)r.ret;
		else if ((hb.comp != UINT64_MAX && r.in_used != hb.comp) || (hb.uncomp != UINT64_MAX && r.out_used != hb.uncomp)) ret = XZB_DATA_ERROR;
		uint64_t p = blks[b].hdr_off + hb.hsize + r.in_used;
		uint64_t c = r.in_used;
		while (ret == XZB_OK && (c & 3)) {
			if (p >= s.in_size) ret = XZB_BUF_ERROR;
			else if (in[p++] != 0x00) ret = XZB_DATA_ERROR;
			++c;
		}
		if (ret == XZB_OK && s.in_size - p < s.csize) ret = XZB_BUF_ERROR;
		if (ret == XZB_OK && cmp)
			for (uint32_t i = 0; i < s.csize; ++i)
				if (chk[(size_t)b * chk_stride + i] != in[p + i]) { ret = XZB_DATA_ERROR; break; }
		if (ret == XZB_OK && s.n_recs >= rec_cap) ret = XZB_PROG_ERROR;  // the caller's record area is too small
		s.ret = ret;
		if (ret != XZB_OK) { s.op = op_fail; break; }
		p += s.csize;
		recs[s.n_recs].unpadded_size = hb.hsize + r.in_used + s.csize;
		recs[s.n_recs].uncompressed_size = r.out_used;
		++s.n_recs;
		s.ip = p; s.op = blks[b].out_off + r.out_used;
		produced += r.out_used;
	}
	if (s.ret == XZB_OK && s.pending != XZB_OK && s.ip == s.bip) s.ret = s.pending;
	if (s.ret != XZB_OK || s.at_index) xzb_dec_end(s, in, crc32_table, recs);
	s.nb = 0;
	return produced;
}

// Index records an item of in_size bytes can produce: every Block takes at least 16 bytes (a 12-byte header, then
// Compressed Data of at least one byte, padded to four).
XZB_HD uint64_t xzb_dec_rec_bound(uint64_t in_size) { return in_size / 16 + 1; }
