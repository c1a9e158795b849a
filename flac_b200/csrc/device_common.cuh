// device_common.cuh -- device helpers shared by every kernel translation unit of libflac_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "fb200_internal.h"
#include "glibc_log_data.h"

namespace fb200 {

#ifndef M_LN2
#define M_LN2 0.69314718055994530942
#endif

// ---------------------------------------------------------------- small helpers

__device__ __forceinline__ uint32_t ilog2_u32(uint32_t v) { return 31u - (uint32_t)__clz((int)v); }
__device__ __forceinline__ uint32_t ilog2_u64(uint64_t v) { return 63u - (uint32_t)__clzll((long long)v); }

// bitmath.c:63-73 FLAC__bitmath_silog2
__device__ __forceinline__ uint32_t silog2_i64(int64_t v)
{
	if(v == 0) return 0;
	if(v == -1) return 2;
	v = (v < 0) ? (-(v + 1)) : v;
	return ilog2_u64((uint64_t)v) + 2;
}

__device__ __forceinline__ uint32_t warp_or(uint32_t v) { return __reduce_or_sync(0xffffffffu, v); }
__device__ __forceinline__ uint32_t warp_and(uint32_t v) { return __reduce_and_sync(0xffffffffu, v); }

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v)
{
#pragma unroll
	for(int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}

__device__ __forceinline__ uint32_t abs_u32(int32_t r) { return r < 0 ? (uint32_t)0 - (uint32_t)r : (uint32_t)r; }

// ================================================================ log()
// The reference calls the HOST libm's log() on its decision path (lpc.c:1594 order guess and
// "don't even try" tests, fixed.c:284-288). CUDA's log() is not bit-identical to glibc's, so this is an
// operation-by-operation restatement of the routine glibc selects on x86-64 hosts with FMA+AVX2
// (`__log_fma`, the FMA build of sysdeps/ieee754/dbl-64/e_log.c), transcribed from its disassembly:
// the same fused and unfused operations in the same order, tables extracted from the same binary
// (glibc_log_data.h). tests/test_gpu_log.py compares it with the host's log() bit for bit.
__device__ __forceinline__ double fb_log(double x)
{
	unsigned long long ix = (unsigned long long)__double_as_longlong(x);
	if(ix - 0x3fee000000000000ull <= 0x308ffffffffffull) {
		// 1 - 2^-4 <= x < 1 + 0x1.09p-4: polynomial in r = x - 1 with a double-double head
		if(ix == 0x3ff0000000000000ull) return 0.0;
		const double r = __dsub_rn(x, 1.0);
		double p2 = __fma_rn(r, kLogB[2], kLogB[1]);
		double p3 = __fma_rn(r, kLogB[5], kLogB[4]);
		const double r2 = __dmul_rn(r, r);
		double p5 = __fma_rn(r, kLogB[8], kLogB[7]);
		p2 = __fma_rn(r2, kLogB[3], p2);
		p3 = __fma_rn(r2, kLogB[6], p3);
		const double r3 = __dmul_rn(r, r2);
		double p1 = __fma_rn(r2, kLogB[9], p5);
		p1 = __fma_rn(r3, kLogB[10], p1);
		p1 = __fma_rn(p1, r3, p3);
		p1 = __fma_rn(p1, r3, p2);
		const double t = __fma_rn(r, 134217728.0, r);        // r + r*2^27
		const double rhi = __fma_rn(-134217728.0, r, t);     // ... - r*2^27
		const double b0 = kLogB[0];
		const double rhi2 = __dmul_rn(rhi, rhi);
		const double rlo = __dsub_rn(r, rhi);
		const double hi = __fma_rn(rhi2, b0, r);
		const double d = __dsub_rn(r, hi);
		const double rs = __dadd_rn(r, rhi);
		double lo = __fma_rn(rhi2, b0, d);
		const double brlo = __dmul_rn(b0, rlo);
		lo = __fma_rn(brlo, rs, lo);
		const double y = __fma_rn(p1, r3, lo);
		return __dadd_rn(hi, y);
	}
	const unsigned int top = (unsigned int)(ix >> 48);
	if(top - 0x10u > 0x7fdfu) {
		// x <= 0, subnormal, inf or nan
		if((ix << 1) == 0) return -CUDART_INF;
		if(ix == 0x7ff0000000000000ull) return x;
		if((top & 0x8000u) || (top & 0x7ff0u) == 0x7ff0u) return CUDART_NAN;
		x = __dmul_rn(x, 4503599627370496.0);  // subnormal: scale by 2^52
		ix = (unsigned long long)__double_as_longlong(x) - (52ull << 52);
	}
	const unsigned long long tmp = ix - 0x3fe6000000000000ull;
	const int i = (int)((tmp >> 45) & 0x7f);
	const int k = (int)((long long)tmp >> 52);
	const unsigned long long iz = ix - (tmp & 0xfff0000000000000ull);
	const double invc = kLogTab[2 * i], logc = kLogTab[2 * i + 1];
	const double z = __longlong_as_double((long long)iz);
	const double kd = (double)k;
	const double w = __fma_rn(kd, kLogLn2Hi, logc);
	const double r = __fma_rn(z, invc, -1.0);
	const double q21 = __fma_rn(r, kLogA[2], kLogA[1]);
	const double hi = __dadd_rn(r, w);
	const double r2 = __dmul_rn(r, r);
	double lo = __dsub_rn(w, hi);
	lo = __dadd_rn(lo, r);
	lo = __fma_rn(kd, kLogLn2Lo, lo);
	const double r3 = __dmul_rn(r, r2);
	double q = __fma_rn(r, kLogA[4], kLogA[3]);
	lo = __fma_rn(r2, kLogA[0], lo);
	q = __fma_rn(q, r2, q21);
	const double y = __fma_rn(r3, q, lo);
	return __dadd_rn(y, hi);
}


// stream_encoder.c:4929-4951 count_rice_bits_in_partition_
__device__ __forceinline__ uint32_t count_rice_bits(uint32_t k, uint32_t partition_samples, uint64_t abs_sum)
{
	const uint64_t v = (uint64_t)kRiceParamLen + (uint64_t)(1 + k) * partition_samples +
	                   (k ? (abs_sum >> (k - 1)) : (abs_sum << 1)) - (partition_samples >> 1);
	return (uint32_t)(v < 0xffffffffull ? v : 0xffffffffull);
}

struct BitPut {
	uint32_t *words;
	uint32_t cur;
	uint32_t pos;
	int widx, first;
	__device__ __forceinline__ void init(uint32_t *w, uint32_t bitpos)
	{
		words = w; pos = bitpos; widx = (int)(bitpos >> 5); first = widx; cur = 0;
	}
	__device__ __forceinline__ void flush()
	{
		if(cur) {
			if(widx == first) atomicOr(&words[widx], cur);
			else words[widx] = cur;  // interior word: exclusively ours, buffer pre-zeroed
		}
		cur = 0;
	}
	__device__ __forceinline__ void skip(uint32_t n)  // n zero bits
	{
		pos += n;
		const int nw = (int)(pos >> 5);
		if(nw != widx) { flush(); widx = nw; }
	}
	__device__ __forceinline__ void put(uint32_t value, uint32_t nbits)  // 1..32 bits, value < 2^nbits
	{
		const uint32_t off = pos & 31u;
		const unsigned long long v = (unsigned long long)value << (64u - off - nbits);
		cur |= (uint32_t)(v >> 32);
		pos += nbits;
		if(off + nbits >= 32u) {
			flush();
			widx++;
			cur = (uint32_t)v;
		}
	}
	__device__ __forceinline__ void finish()
	{
		if(cur) atomicOr(&words[widx], cur);  // last (partial) word may be shared
		cur = 0;
	}
};

__device__ __forceinline__ uint32_t mask_bits(int32_t v, uint32_t n) { return n >= 32 ? (uint32_t)v : ((uint32_t)v & ((1u << n) - 1u)); }
__device__ __forceinline__ int skew(int i) { return i + (i >> 5); }  // bank-conflict-free run access

// GF(2)[x] multiply mod x^16+x^15+x^2+1 (CRC-16 poly 0x8005, crc.c:78)
__device__ __forceinline__ uint32_t gf16_mul(uint32_t a, uint32_t b)
{
	uint32_t r = 0;
#pragma unroll
	for(int i = 15; i >= 0; i--) {
		r = (r & 0x8000u) ? ((r << 1) ^ 0x8005u) & 0xffffu : (r << 1);
		if((b >> i) & 1u) r ^= a;
	}
	return r;
}

// x^(2^j) mod (x^16+x^15+x^2+1) for j = 0..14 (x has order 32767, so x^(2^15) = x and the table is periodic);
// generated with gf16_mul by repeated squaring from x = 0x2.
__device__ __constant__ const uint16_t kCrcXPow2[15] = {0x2, 0x4, 0x10, 0x100, 0x8005, 0x8017, 0x8113, 0x106, 0x8011, 0x8107, 0x16, 0x114, 0x8115, 0x112, 0x8101};

// x^(8k) mod (x^8+x^2+x+1), k = 0..15: weights that combine per-byte CRC-8s of a frame header (crc.c:39-76)
__device__ __constant__ const uint8_t kCrc8XPow8[16] = {0x01, 0x07, 0x15, 0x6b, 0x16, 0x62, 0x29, 0xdf, 0x13, 0x79, 0x68, 0x1f, 0x5d, 0x94, 0xe5, 0xb5};

// fixed predictors as FIR taps (fixed.c:470-530): r = x[i] - sum_j c[j] x[i-1-j]
__device__ __forceinline__ int fixed_tap(int order, int j)
{
	// order 1: {1}; 2: {2,-1}; 3: {3,-3,1}; 4: {4,-6,4,-1}
	const int tab[5][4] = {{0, 0, 0, 0}, {1, 0, 0, 0}, {2, -1, 0, 0}, {3, -3, 1, 0}, {4, -6, 4, -1}};
	return j < 4 ? tab[order][j] : 0;
}

// |residual| sum of G consecutive outputs. xg[MAXORD + m] = output sample m, xg[0..MAXORD) = history.
// MASKED: leave out the first ord0 outputs (the warm-up samples of the block's very first group;
// order <= MAXORD <= ... so only outputs m < MAXORD can be masked).
// The body is deliberately small (G x NTAPS MACs): the callers loop over groups with a ROLLED loop so
// the hot code stays inside the instruction cache (a fully unrolled 32 x 12 run per variant did not: the
// profiler showed warps stalled on instruction fetch).
template <int G, int MAXORD, int NTAPS, bool WIDE, bool MASKED, bool NARROW>
__device__ __forceinline__ void group_abs_sum(const int (&xg)[MAXORD + G], const int (&q)[MAXORD], int shift, int ord0, int limit,
                                              uint32_t &s32, unsigned long long &s64, bool &bad)
{
	constexpr bool narrow_acc = NARROW;
#pragma unroll
	for(int m = 0; m < G; m++) {
		uint32_t a;
		bool keep = true;
		if(MASKED && m < MAXORD) keep = m >= ord0;
		if(!WIDE) {
			int sum = 0;
#pragma unroll
			for(int j = 0; j < NTAPS; j++) sum += q[j] * xg[MAXORD + m - 1 - j];
			const int pred = sum >> shift;
			if(narrow_acc && !(MASKED && m < MAXORD)) { s32 = __sad(xg[MAXORD + m], pred, s32); continue; }
			a = __sad(xg[MAXORD + m], pred, 0u);
		}
		else {
			long long sum = 0;
#pragma unroll
			for(int j = 0; j < NTAPS; j++) sum += (long long)q[j] * (long long)xg[MAXORD + m - 1 - j];
			const long long rr = (long long)xg[MAXORD + m] - (sum >> shift);
			if(limit && (rr <= (long long)INT32_MIN || rr > (long long)INT32_MAX)) bad = true;  // lpc.c:868-884
			a = abs_u32((int)rr);
		}
		if(keep) { if(narrow_acc) s32 += a; else s64 += a; }
	}
}


// int32 -> double without the conversion pipe: the bit pattern 0x43300000:(x ^ 0x80000000) is 2^52 + 2^31 + x.
__device__ __forceinline__ double int_to_double_exact(int x)
{
	return __dsub_rn(__hiloint2double(0x43300000, (int)((unsigned)x ^ 0x80000000u)), 4503601774854144.0);
}

// ---------------------------------------------------------------- TMA (1-D bulk copy) + mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{
	const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes)
{
	const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(a), "r"(bytes) : "memory");
}
// global -> shared bulk copy, completion counted in bytes on `bar`. size % 16 == 0, both addresses 16-byte aligned.
__device__ __forceinline__ void tma_bulk_g2s(void *smem_dst, const void *gmem_src, unsigned bytes, uint64_t *bar)
{
	const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
	const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(d), "l"(gmem_src), "r"(bytes), "r"(b)
	             : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{
	const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
	asm volatile(
	    "{\n"
	    ".reg .pred p;\n"
	    "WAIT_%=:\n"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
	    "@p bra DONE_%=;\n"
	    "bra WAIT_%=;\n"
	    "DONE_%=:\n"
	    "}\n" ::"r"(a),
	    "r"(parity)
	    : "memory");
}


}  // namespace fb200
