// xzb_sha256.cuh -- SHA-256 (FIPS 180-4) of one buffer, host/device, for the .xz Check field
// (LZMA_CHECK_SHA256 = 10, 32 bytes; reference: check/sha256.c, check/check.c:97-174).
// One thread hashes one .xz block: the compression function is a serial chain per message, so
// the kernel (xzb_k_sha256) gets its parallelism from the blocks of a wave and runs on the SMs
// the parser kernel leaves idle.
#pragma once
#include "xzb_common.cuh"

#ifdef __CUDA_ARCH__
#define XZB_SHA_CONST __constant__
#else
#define XZB_SHA_CONST static
#endif

XZB_SHA_CONST const uint32_t xzb_sha256_k[64] = {
	0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
	0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
	0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
	0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
	0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
	0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
	0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
	0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u };

XZB_HD uint32_t xzb_rotr32(uint32_t x, uint32_t n) { return (x >> n) | (x << (32 - n)); }

// one 64-byte chunk given as 16 big-endian words
XZB_HD void xzb_sha256_compress(uint32_t h[8], uint32_t w[16])
{
	uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
	for (uint32_t t = 0; t < 64; ++t) {
		if (t >= 16) {  // message schedule in a 16-word ring
			const uint32_t w15 = w[(t + 1) & 15], w2 = w[(t + 14) & 15];
			const uint32_t s0 = xzb_rotr32(w15, 7) ^ xzb_rotr32(w15, 18) ^ (w15 >> 3);
			const uint32_t s1 = xzb_rotr32(w2, 17) ^ xzb_rotr32(w2, 19) ^ (w2 >> 10);
			w[t & 15] += s0 + w[(t + 9) & 15] + s1;
		}
		const uint32_t S1 = xzb_rotr32(e, 6) ^ xzb_rotr32(e, 11) ^ xzb_rotr32(e, 25);
		const uint32_t ch = (e & f) ^ (~e & g);
		const uint32_t t1 = hh + S1 + ch + xzb_sha256_k[t] + w[t & 15];
		const uint32_t S0 = xzb_rotr32(a, 2) ^ xzb_rotr32(a, 13) ^ xzb_rotr32(a, 22);
		const uint32_t maj = (a & b) ^ (a & c) ^ (b & c);
		const uint32_t t2 = S0 + maj;
		hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
	}
	h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

XZB_HD uint32_t xzb_be32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

XZB_HD void xzb_sha256(const uint8_t *data, uint32_t size, uint8_t out[32])
{
	uint32_t h[8] = { 0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u };
	uint32_t w[16];
	uint32_t pos = 0;
	for (; size - pos >= 64; pos += 64) {
		for (int i = 0; i < 16; ++i) w[i] = xzb_be32(data + pos + 4 * i);
		xzb_sha256_compress(h, w);
	}
	// padding: 0x80, zeros, 64-bit big-endian bit count (one or two more chunks)
	uint8_t tail[128];
	const uint32_t rem = size - pos;
	for (uint32_t i = 0; i < rem; ++i) tail[i] = data[pos + i];
	tail[rem] = 0x80;
	const uint32_t total = rem + 1 + 8 <= 64 ? 64u : 128u;
	for (uint32_t i = rem + 1; i < total - 8; ++i) tail[i] = 0;
	const uint64_t bits = (uint64_t)size * 8;
	for (int i = 0; i < 8; ++i) tail[total - 1 - i] = (uint8_t)(bits >> (8 * i));
	for (uint32_t c = 0; c < total; c += 64) {
		for (int i = 0; i < 16; ++i) w[i] = xzb_be32(tail + c + 4 * i);
		xzb_sha256_compress(h, w);
	}
	for (int i = 0; i < 8; ++i) { out[4 * i] = (uint8_t)(h[i] >> 24); out[4 * i + 1] = (uint8_t)(h[i] >> 16); out[4 * i + 2] = (uint8_t)(h[i] >> 8); out[4 * i + 3] = (uint8_t)h[i]; }
}

// The same hash over a message that arrives in pieces (a Block decoded chunk run by chunk run): the chaining value,
// the byte count and the partial 64-byte block live in a plain struct that can sit in device memory between calls.
struct XzbSha256State {
	uint32_t h[8];
	uint64_t count;      // bytes hashed so far
	uint8_t buf[64];     // the partial block: count % 64 bytes
};
XZB_HD void xzb_sha256_init(XzbSha256State *s)
{
	const uint32_t iv[8] = { 0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u };
	for (int i = 0; i < 8; ++i) s->h[i] = iv[i];
	s->count = 0;
}
XZB_HD void xzb_sha256_update(XzbSha256State *s, const uint8_t *data, uint64_t size)
{
	uint32_t w[16];
	uint32_t have = (uint32_t)(s->count & 63);
	s->count += size;
	uint64_t pos = 0;
	if (have) {
		while (have < 64 && pos < size) s->buf[have++] = data[pos++];
		if (have < 64) return;
		for (int i = 0; i < 16; ++i) w[i] = xzb_be32(s->buf + 4 * i);
		xzb_sha256_compress(s->h, w);
	}
	for (; size - pos >= 64; pos += 64) {
		for (int i = 0; i < 16; ++i) w[i] = xzb_be32(data + pos + 4 * i);
		xzb_sha256_compress(s->h, w);
	}
	for (uint32_t i = 0; pos < size; ++i) s->buf[i] = data[pos++];
}
XZB_HD void xzb_sha256_final(XzbSha256State *s, uint8_t out[32])
{
	uint32_t w[16];
	uint8_t tail[128];
	const uint32_t rem = (uint32_t)(s->count & 63);
	for (uint32_t i = 0; i < rem; ++i) tail[i] = s->buf[i];
	tail[rem] = 0x80;
	const uint32_t total = rem + 1 + 8 <= 64 ? 64u : 128u;
	for (uint32_t i = rem + 1; i < total - 8; ++i) tail[i] = 0;
	const uint64_t bits = s->count * 8;
	for (int i = 0; i < 8; ++i) tail[total - 1 - i] = (uint8_t)(bits >> (8 * i));
	for (uint32_t c = 0; c < total; c += 64) {
		for (int i = 0; i < 16; ++i) w[i] = xzb_be32(tail + c + 4 * i);
		xzb_sha256_compress(s->h, w);
	}
	for (int i = 0; i < 8; ++i) { out[4 * i] = (uint8_t)(s->h[i] >> 24); out[4 * i + 1] = (uint8_t)(s->h[i] >> 16); out[4 * i + 2] = (uint8_t)(s->h[i] >> 8); out[4 * i + 3] = (uint8_t)s->h[i]; }
}
