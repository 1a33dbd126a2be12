// xzb_params.h -- host-side derivation of the per-filter constants (XzbParams) from LZMA2
// options, and the table generators.  Reference: lz/lz_encoder.c:191-368 (lz_encoder_prepare),
// lzma/lzma_encoder.c:453-707 (is_options_valid, set_lz_options, lzma_lzma_encoder_create),
// lzma/lzma_encoder_presets.c:16-63, check/crc32_tablegen.c, check/crc64_tablegen.c,
// rangecoder/price_tablegen.c:28-56.
#pragma once
#include <algorithm>
#include <vector>

#include "xzb_common.cuh"
#include "xzb_frame.cuh"

struct XzbLzmaOptions {  // the subset of lzma_options_lzma (api/lzma/lzma12.h:216-525) on the path
	uint32_t dict_size, lc, lp, pb, mode, nice_len, mf, depth;
};

static inline int xzb_preset(XzbLzmaOptions *o, uint32_t preset)  // lzma_lzma_preset
{
	const uint32_t level = preset & 0x1F, flags = preset & ~0x1Fu;
	if (level > 9 || (flags & ~0x80000000u)) return 1;
	static const uint8_t dict_pow2[] = { 18, 20, 21, 22, 22, 23, 23, 24, 25, 26 };
	o->lc = 3; o->lp = 0; o->pb = 2;
	o->dict_size = 1u << dict_pow2[level];
	if (level <= 3) {
		static const uint8_t depths[] = { 4, 8, 24, 48 };
		o->mode = XZB_MODE_FAST;
		o->mf = level == 0 ? XZB_MF_HC3 : XZB_MF_HC4;
		o->nice_len = level <= 1 ? 128 : 273;
		o->depth = depths[level];
	} else {
		o->mode = XZB_MODE_NORMAL;
		o->mf = XZB_MF_BT4;
		o->nice_len = level == 4 ? 16 : level == 5 ? 32 : 64;
		o->depth = 0;
	}
	if (flags & 0x80000000u) {
		o->mode = XZB_MODE_NORMAL;
		o->mf = XZB_MF_BT4;
		if (level == 3 || level == 5) { o->nice_len = 192; o->depth = 0; }
		else { o->nice_len = 273; o->depth = 512; }
	}
	return 0;
}

// Returns XZB_OK or XZB_OPTIONS_ERROR (same validation as the reference's init chain).
static inline int xzb_make_params(const XzbLzmaOptions *o, XzbParams *P)
{
	if (o->lc > 4 || o->lp > 4 || o->lc + o->lp > 4 || o->pb > 4) return XZB_OPTIONS_ERROR;
	if (o->nice_len < XZB_MATCH_LEN_MIN || o->nice_len > XZB_MATCH_LEN_MAX) return XZB_OPTIONS_ERROR;
	if (o->mode != XZB_MODE_FAST && o->mode != XZB_MODE_NORMAL) return XZB_OPTIONS_ERROR;
	if (o->mf != XZB_MF_HC3 && o->mf != XZB_MF_HC4 && o->mf != XZB_MF_BT2 && o->mf != XZB_MF_BT3 && o->mf != XZB_MF_BT4) return XZB_OPTIONS_ERROR;
	// IS_ENC_DICT_SIZE_VALID, lz/lz_encoder.h:22-26: 4 KiB .. 1.5 GiB
	if (o->dict_size < 4096 || o->dict_size > (1u << 30) + (1u << 29)) return XZB_OPTIONS_ERROR;
	P->dict_size = o->dict_size; P->lc = o->lc; P->lp = o->lp; P->pb = o->pb; P->mode = o->mode; P->mf = o->mf;
	P->hash_bytes = o->mf & 0x0F; P->is_bt = (o->mf & 0x10) != 0;
	P->nice_len = o->nice_len > P->hash_bytes ? o->nice_len : P->hash_bytes;
	P->cyclic_size = o->dict_size + 1;
	uint32_t hs;
	if (P->hash_bytes == 2) {
		hs = 0xFFFF;
	} else {
		hs = o->dict_size - 1;
		hs |= hs >> 1; hs |= hs >> 2; hs |= hs >> 4; hs |= hs >> 8;
		hs >>= 1; hs |= 0xFFFF;
		if (hs > (1u << 24)) { if (P->hash_bytes == 3) hs = (1u << 24) - 1; else hs >>= 1; }
	}
	P->hash_mask = hs;
	P->depth = o->depth;
	if (P->depth == 0) P->depth = P->is_bt ? 16 + P->nice_len / 2 : 4 + P->nice_len / 4;
	uint32_t log_size = 0;
	while ((1u << log_size) < o->dict_size) ++log_size;
	P->dist_table_size = log_size * 2;
	P->len_table_size = P->nice_len + 1 - XZB_MATCH_LEN_MIN;
	P->mstride = 8;
	P->dict_prop = xzb_lzma2_dict_prop(o->dict_size);
	P->lclppb = (uint8_t)((o->pb * 5 + o->lp) * 9 + o->lc);
	P->n_pre = 0; P->ff_len = 0;
	return XZB_OK;
}

// ---- wave layout and planning (host) ----
// A wave is B Blocks resident in HBM side by side.  Block b's positions start at off[b] in every per-position array
// (keys, prev*, son, mh, mp, ovf); each start is a multiple of XZB_WAVE_ALIGN positions, so a 256-position tile of the
// match-finder launches belongs to exactly one Block and no cache line of mh / mp holds two Blocks' rows.
#define XZB_WAVE_ALIGN 256u

static inline uint64_t xzb_wave_pad(uint64_t n) { return (n + XZB_WAVE_ALIGN - 1) & ~(uint64_t)(XZB_WAVE_ALIGN - 1); }

// Scratch a Block of n bytes is coded into (header + LZMA2 data + padding + check, with room to spare).
static inline uint32_t xzb_scratch_cap(uint64_t n) { return (uint32_t)(n + n / 4096 + 70000 + 1024) & ~15u; }

// Workspace of one Block: per_byte for each (padded) position, per_block on top of that.
struct XzbWaveCost { uint64_t per_byte, per_block; };
static inline XzbWaveCost xzb_wave_cost(const XzbParams &P)
{
	// keys, vals (two each), prev2/3/m, mh, ovf, mp; BT adds son and the run lists; scratch; in- and output staging
	const uint64_t per_byte = 16 + 8 + 12 + 8 + 4 + 8 * (uint64_t)P.mstride + 8 + (P.is_bt ? 16 : 0) + 2 + 2;
	return XzbWaveCost{ per_byte, 70000 + 1024 + 4096 + 256 };
}

// Batch wave planner.  Items (sizes[i] > 0) are taken largest first (ties in index order), so a wave holds similar
// sizes and its longest serial chains are dispatched first; a wave takes items while all of these hold:
//   cost.per_byte * sum(padded n) + cost.per_block * B <= budget  (a wave always takes at least one item),
//   (B << hash_bits) < 2^32  (the sort keys are (block << hash_bits) | hash),
//   sum(padded n) < 2^32 - 16,  B <= max_blocks (0: no limit).
// order: item indices in wave order; wave_start: index into `order` where each wave begins, plus order.size().
static inline void xzb_plan_waves(const uint64_t *sizes, uint32_t n, XzbWaveCost cost, uint64_t budget, uint32_t hash_bits,
		uint32_t max_blocks, std::vector<uint32_t> *order, std::vector<uint32_t> *wave_start)
{
	order->resize(n);
	for (uint32_t i = 0; i < n; ++i) (*order)[i] = i;
	std::stable_sort(order->begin(), order->end(), [&](uint32_t a, uint32_t b) { return sizes[a] > sizes[b]; });
	const uint64_t key_cap = (1ull << (32 - hash_bits)) - 1;
	wave_start->clear();
	uint64_t B = 0, pos = 0;
	for (uint32_t k = 0; k < n; ++k) {
		const uint64_t np = xzb_wave_pad(sizes[(*order)[k]]);
		const bool fits = B > 0 && B + 1 <= key_cap && (max_blocks == 0 || B + 1 <= max_blocks) && pos + np < 0xFFFFFFF0ull
			&& cost.per_byte * (pos + np) + cost.per_block * (B + 1) <= budget;
		if (!fits) { wave_start->push_back(k); B = 0; pos = 0; }
		++B; pos += np;
	}
	wave_start->push_back(n);
}

// Start of each Block's positions in a wave of Blocks of sizes n[0..B): the padded sizes summed.  Returns the total.
static inline uint64_t xzb_wave_offsets(const uint32_t *n, uint32_t B, uint32_t *off)
{
	uint64_t pos = 0;
	for (uint32_t b = 0; b < B; ++b) { off[b] = (uint32_t)pos; pos += xzb_wave_pad(n[b]); }
	return pos;
}

// Groups of the device-resident Stream decoder (xzb_stream_buffer_decode_batch_device): items in call order, item i
// costing per_item + 16 * (in_size[i] / 16 + 1) bytes of HBM (its cursor and its Index record area, xzb_dec_rec_bound);
// a group takes items while their sum stays within budget, and always at least one.  group_start: the first item of
// each group, plus n.
static inline void xzb_plan_dec_groups(const uint64_t *in_size, uint32_t n, uint64_t per_item, uint64_t budget, std::vector<uint32_t> *group_start)
{
	group_start->clear();
	uint64_t used = 0;
	for (uint32_t i = 0; i < n; ++i) {
		const uint64_t c = per_item + 16 * (in_size[i] / 16 + 1);
		if (i == 0 || used + c > budget) { group_start->push_back(i); used = 0; }
		used += c;
	}
	group_start->push_back(n);
}

struct XzbHostTables { uint32_t crc32[256]; uint64_t crc64[256]; uint8_t prices[128]; };

static inline void xzb_make_tables(XzbHostTables *t)
{
	for (uint32_t b = 0; b < 256; ++b) {
		uint32_t r = b;
		for (int i = 0; i < 8; ++i) r = (r & 1) ? (r >> 1) ^ 0xEDB88320u : r >> 1;
		t->crc32[b] = r;
		uint64_t q = b;
		for (int i = 0; i < 8; ++i) q = (q & 1) ? (q >> 1) ^ 0xC96C5795D7870F42ull : q >> 1;
		t->crc64[b] = q;
	}
	for (uint32_t i = 8; i < 2048; i += 16) {
		uint32_t w = i, bit_count = 0;
		for (int j = 0; j < 4; ++j) {
			w *= w; bit_count <<= 1;
			while (w >= (1u << 16)) { w >>= 1; ++bit_count; }
		}
		t->prices[i >> 4] = (uint8_t)((11 << 4) - 15 - bit_count);
	}
}
