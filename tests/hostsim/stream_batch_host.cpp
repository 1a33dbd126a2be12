// tests/hostsim/stream_batch_host.cpp -- TEST HARNESS (tests only): the whole-Stream batch encoder's host pieces
// compiled with g++ so that tests/test_stream_batch_cpu.py can drive them on a box without a GPU: Stream placement
// (xzb_stream_place) and the multi-Block Stream packing that xzb_k_pack_streams runs (xzb_pack_block, xzb_frame.cuh).
// Not part of the product and never used as a fallback.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../xz_b200/csrc/xzb_common.cuh"
#include "../../xz_b200/csrc/xzb_frame.cuh"
#include "../../xz_b200/csrc/xzb_params.h"

extern "C" {

// Whole Streams rebuilt from their finished Blocks as the batch driver places them: item i's Stream has nblocks[i]
// Blocks and goes to out + out_off[i] (room out_cap[i]).  Block k (in (item, j) order) is blocks[boff[k] .. + bsize[k])
// with its Index record (unpadded[k], uncomp[k]); wave[k] is the wave it finishes in.  Wave by wave, each Block is placed
// with xzb_stream_place and packed with xzb_pack_block, work-shared by `nthreads` workers run one after another; the
// Streams with no Block come last.  ret[i] = 0 or XZB_BUF_ERROR, out_size[i] the Stream's size.  Returns the waves run.
uint32_t bh_pack_waves(uint32_t n, const uint64_t *nblocks, const uint8_t *blocks, const uint64_t *boff, const uint32_t *bsize,
		const uint64_t *unpadded, const uint64_t *uncomp, const uint32_t *wave, uint32_t check, uint32_t nthreads,
		uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_size, uint32_t *ret)
{
	static XzbHostTables tab;
	static bool init = false;
	if (!init) { xzb_make_tables(&tab); init = true; }
	std::vector<XzbStreamPlace> place(n);
	std::vector<uint32_t> item, j;
	for (uint32_t i = 0; i < n; ++i) {
		place[i].cap = out_cap[i]; place[i].nblocks = nblocks[i];
		out_size[i] = 0; ret[i] = XZB_OK;
		for (uint64_t b = 0; b < nblocks[i]; ++b) { item.push_back(i); j.push_back((uint32_t)b); }
	}
	uint32_t waves = 0;
	for (size_t k = 0; k < item.size(); ++k) waves = std::max(waves, wave[k] + 1);
	auto pack = [&](uint32_t i, uint64_t at, uint32_t flags, const uint8_t *src, uint32_t size) {
		std::vector<XzbV16> aligned(size / 16 + 1);
		if (size) memcpy(aligned.data(), src, size);
		const XzbStreamPlace &s = place[i];
		for (uint32_t t = 0; t < nthreads; ++t)
			xzb_pack_block(tab.crc32, out + out_off[i] + at, (const uint8_t *)aligned.data(), size, flags, s.recs.data(), s.recs.data() + s.nblocks,
					s.nblocks, check, t, nthreads);
		if (flags & XZB_PACK_TAIL) out_size[i] = s.pos;
	};
	for (uint32_t w = 0; w < waves; ++w)
		for (size_t k = 0; k < item.size(); ++k) {
			const uint32_t i = item[k];
			if (wave[k] != w || ret[i] != XZB_OK) continue;
			if (j[k] != place[i].next) return UINT32_MAX;   // placed out of order
			uint32_t flags;
			const uint64_t at = xzb_stream_place(place[i], bsize[k], unpadded[k], uncomp[k], &flags);
			if (at == UINT64_MAX) { ret[i] = XZB_BUF_ERROR; continue; }
			pack(i, at, flags, blocks + boff[k], bsize[k]);
		}
	for (uint32_t i = 0; i < n; ++i)
		if (nblocks[i] == 0) {
			uint32_t flags;
			const uint64_t at = xzb_stream_place(place[i], 0, 0, 0, &flags);
			if (at == UINT64_MAX) ret[i] = XZB_BUF_ERROR; else pack(i, at, flags, nullptr, 0);
		}
	return waves;
}

}  // extern "C"
