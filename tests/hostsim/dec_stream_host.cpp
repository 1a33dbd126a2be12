// tests/hostsim/dec_stream_host.cpp -- TEST HARNESS (tests only): the device Stream decoder's host pieces compiled with
// g++ so that tests/test_dec_stream_cpu.py can drive them on a box without a GPU: the grouping (xzb_params.h) and the
// round loop of xzb_stream_buffer_decode_batch_device over the Stream step functions (xzb_dec_stream.cuh).  Not part
// of the product and never used as a fallback.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../xz_b200/csrc/xzb_common.cuh"
#include "../../xz_b200/csrc/xzb_frame.cuh"
#include "../../xz_b200/csrc/xzb_params.h"
#include "../../xz_b200/csrc/xzb_dec_stream.cuh"
#include "../../xz_b200/csrc/xzb_filters.cuh"
#include "../../xz_b200/csrc/xzb_sha256.cuh"

extern "C" {

// group[i]: the group of item i under xzb_plan_dec_groups.  Returns the groups.
uint32_t ds_plan_dec_groups(const uint64_t *in_size, uint32_t n, uint64_t per_item, uint64_t budget, uint32_t *group)
{
	std::vector<uint32_t> start;
	xzb_plan_dec_groups(in_size, n, per_item, budget, &start);
	for (size_t g = 0; g + 1 < start.size(); ++g)
		for (uint32_t i = start[g]; i < start[g + 1]; ++i) group[i] = (uint32_t)g;
	return (uint32_t)start.size() - 1;
}

// The round loop of xzb_stream_buffer_decode_batch_device on the CPU: the same step functions, with the host form of
// the LZMA2 decoder (xzb_dec.cuh), the filters (xzb_filters.cuh), CRC and SHA-256 in place of the kernels.  At most
// `cap` Blocks per round, granted to items in call order as the scan kernel's atomicAdd may grant them.  Output goes
// straight into each item's slot.  *rounds: the rounds taken.
int ds_decode_batch(uint32_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_size, uint8_t *out, const uint64_t *out_off,
		const uint64_t *out_cap, uint64_t *out_size, uint64_t *in_used, uint32_t *ret, uint32_t flags, uint32_t cap, uint32_t *rounds)
{
	static XzbHostTables tab;
	static bool init = false;
	if (!init) { xzb_make_tables(&tab); init = true; }
	std::vector<XzbDecCursor> cur(n);
	std::vector<std::vector<xzb_index_record>> recs(n);
	for (uint32_t i = 0; i < n; ++i) { xzb_dec_init(cur[i], in_size[i], out_cap[i], flags, 0); recs[i].resize(xzb_dec_rec_bound(in_size[i])); }
	std::vector<XzbDecBlk> blks(cap);
	std::vector<XzbDecResult> res(cap);
	std::vector<uint8_t> chk(32 * (size_t)cap);
	std::vector<uint32_t> job0(n), nbs(n);
	XzbDec *d = (XzbDec *)malloc(sizeof(XzbDec));
	*rounds = 0;
	for (;;) {
		uint32_t njobs = 0;
		for (uint32_t i = 0; i < n; ++i) {                 // xzb_k_dec_scan
			nbs[i] = 0;
			if (cur[i].done) continue;
			const uint8_t *src = in + in_off[i];
			XzbDecCursor c = cur[i];
			const uint32_t want = xzb_dec_scan(c, src, tab.crc32, nullptr, cap, recs[i].data());
			if (want == 0) { cur[i] = c; continue; }
			const uint32_t base = njobs;
			njobs += want;
			if (base >= cap) continue;
			nbs[i] = xzb_dec_scan(cur[i], src, tab.crc32, blks.data() + base, std::min(want, cap - base), recs[i].data());
			job0[i] = base;
		}
		if (njobs == 0) break;
		++*rounds;
		bool live = false;
		for (uint32_t i = 0; i < n; ++i) {
			if (nbs[i] == 0) { live = live || !cur[i].done; continue; }
			const uint32_t ck = xzb_dec_check_computed(cur[i]);
			for (uint32_t b = 0; b < nbs[i]; ++b) {
				const XzbDecBlk &k = blks[job0[i] + b];
				XzbDecResult &r = res[job0[i] + b];
				uint8_t *o = out + out_off[i] + k.out_off;
				r.ret = (uint32_t)xzb_lzma2_decode(d, in + in_off[i] + k.hdr_off + k.hb.hsize, k.in_avail, k.hb.dict_size, o, k.out_limit,
						&r.in_used, &r.out_used, 0, 1);
				for (uint32_t l = k.hb.n_pre; l-- > 0;) xzb_filter_apply_seq(k.hb.pre[l], o, r.out_used, false);
				uint8_t *cv = chk.data() + 32 * (size_t)(job0[i] + b);
				if (ck == 10) xzb_sha256(o, r.out_used, cv);
				else {
					uint64_t v = 0;
					if (ck == 1) v = xzb_crc32_bytes(tab.crc32, o, r.out_used, 0);
					else if (ck == 4) { uint64_t c = ~0ull; for (uint32_t p = 0; p < r.out_used; ++p) c = tab.crc64[(c ^ o[p]) & 0xFF] ^ (c >> 8); v = ~c; }
					for (int q = 0; q < 8; ++q) cv[q] = (uint8_t)(v >> (8 * q));
				}
			}
			xzb_dec_settle(cur[i], in + in_off[i], tab.crc32, blks.data() + job0[i], res.data() + job0[i], chk.data() + 32 * (size_t)job0[i], 32,
					recs[i].data(), recs[i].size());
			live = live || !cur[i].done;
		}
		if (!live) break;
	}
	free(d);
	for (uint32_t i = 0; i < n; ++i) {
		const XzbDecCursor &c = cur[i];
		ret[i] = (uint32_t)(c.ret == XZB_BUF_ERROR && c.buf_reason == 1 ? XZB_DATA_ERROR : c.ret);
		out_size[i] = c.out_size; in_used[i] = c.in_used;
	}
	return XZB_OK;
}

}  // extern "C"
