// tests/hostsim/batch_host.cpp -- TEST HARNESS (tests only): the batch encoder's host pieces compiled with g++ so that
// tests/test_batch_cpu.py can drive them on a box without a GPU: wave planning and layout (xzb_params.h) and the
// Stream packing that xzb_k_pack_streams runs (xzb_frame.cuh).  Not part of the product and never used as a fallback.
#include <cstring>
#include <vector>

#include "../../xz_b200/csrc/xzb_common.cuh"
#include "../../xz_b200/csrc/xzb_frame.cuh"
#include "../../xz_b200/csrc/xzb_params.h"

extern "C" {

// order[k]: the item placed k-th; wave[k]: its wave; off[k]: its Block's first position in that wave.  Returns the waves.
uint32_t bh_plan_waves(const uint64_t *sizes, uint32_t n, uint64_t per_byte, uint64_t per_block, uint64_t budget, uint32_t hash_bits,
		uint32_t max_blocks, uint32_t *order, uint32_t *wave, uint32_t *off)
{
	std::vector<uint32_t> ord, start;
	xzb_plan_waves(sizes, n, XzbWaveCost{ per_byte, per_block }, budget, hash_bits, max_blocks, &ord, &start);
	for (size_t w = 0; w + 1 < start.size(); ++w) {
		std::vector<uint32_t> wn;
		for (uint32_t k = start[w]; k < start[w + 1]; ++k) { order[k] = ord[k]; wave[k] = (uint32_t)w; wn.push_back((uint32_t)sizes[ord[k]]); }
		xzb_wave_offsets(wn.data(), (uint32_t)wn.size(), off + start[w]);
	}
	return (uint32_t)start.size() - 1;
}

// The one-shot Stream around `block` (copied into 16-byte aligned memory first, as scratch is); returns its size.
uint64_t bh_pack_stream(const uint8_t *block, uint32_t block_size, uint64_t unpadded, uint64_t uncomp, uint32_t check, uint8_t *out)
{
	static XzbHostTables tab;
	static bool init = false;
	if (!init) { xzb_make_tables(&tab); init = true; }
	std::vector<XzbV16> aligned(block_size / 16 + 1);
	if (block_size) memcpy(aligned.data(), block, block_size);
	return xzb_pack_stream(tab.crc32, out, (const uint8_t *)aligned.data(), block_size, unpadded, uncomp, check, true, 0, 1);
}

}  // extern "C"
