// device_common.cuh -- device helpers shared by every kernel translation unit of libflac_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "fb200_internal.h"
#include "flac_frame.cuh"
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

// ---------------------------------------------------------------- search / emit pieces shared by k_search / k_emit and the
// tiled kernels (tiled_kernels.cu)

// fixed.c:222-290 FLAC__fixed_compute_best_predictor: from the abs sums t[k] of the k-th differences over samples 4..bs-1,
// the guessed order and every order's residual bits per sample
__device__ __forceinline__ int fixed_best_order(const unsigned long long (&t)[5], int bs, float (&rbps)[5])
{
	int guess;
	const unsigned long long m34 = t[3] < t[4] ? t[3] : t[4], m234 = t[2] < m34 ? t[2] : m34, m1234 = t[1] < m234 ? t[1] : m234;
	if(t[0] <= m1234) guess = 0;
	else if(t[1] <= m234) guess = 1;
	else if(t[2] <= m34) guess = 2;
	else if(t[3] <= t[4]) guess = 3;
	else guess = 4;
	const double n = (double)(uint32_t)(bs - (int)kMaxFixedOrder);
#pragma unroll
	for(int k = 0; k < 5; k++)
		rbps[k] = (float)((t[k] > 0) ? fb_log(M_LN2 * (double)t[k] / n) / M_LN2 : 0.0);
	return guess;
}

// stream_encoder.c:4098-4103: the fixed order of a subframe is guessed by the _wide routine, the one libFLAC replaces with its
// AVX2 version on x86-64 hosts that have AVX2. With EncK::x86_avx2_fixed_guess set, such subframes take that version's sums.
__device__ __forceinline__ bool fixed_guess_avx2(const EncK &P, int bs, int sbps)
{
	return P.x86_avx2_fixed_guess && sbps < 28 && sbps + (int)ilog2_u32((uint32_t)(bs - (int)kMaxFixedOrder) * 17u) >= 32;
}

// Turns the C routine's fixed-guess sums into the x86 AVX2 routine's. te holds fixed.c:222-290's abs sums of the 0th .. 4th
// differences over samples 4 .. bs-1 of the block x; afterwards it holds those of FLAC__fixed_compute_best_predictor_wide_intrin_avx2
// (fixed_intrin_avx2.c:57-138). That routine splits the n = bs - 4 positions past the warm-up into four lanes: lane j = 0..3 sums
// q = n / 4 positions from od_j = (j n) / 4 on, with positions op_j - 4 .. op_j - 1 (op_j = j q) as its difference history.
// When n % 4 == 0 the two agree. Otherwise the n % 4 positions between two lanes and behind lane 3 are not summed, and the
// first four positions of a lane whose history lies od_j - op_j (1 or 2) samples further back take their differences against
// that history. So one thread corrects the sums by at most 11 positions' terms; they wrap on the way but end exact.
__device__ __forceinline__ void fixed_guess_avx2_fixup(const int32_t *x, int bs, unsigned long long *te)
{
	const int n = bs - (int)kMaxFixedOrder, q = n >> 2;
	if((n & 3) == 0) return;
	const int32_t *d = x + kMaxFixedOrder;  // position p is d[p]
	// adds (sign 1) or removes (sign -1) position p's terms; its predecessors m > k lie `back` samples further back. Subframe
	// samples have at most 25 bits here (24-bit side channels), so every difference fits 32 bits.
	auto terms = [&](int p, int k, int back, unsigned long long sign) {
		const int32_t d0 = d[p], d1 = d[k < 1 ? p - 1 - back : p - 1], d2 = d[k < 2 ? p - 2 - back : p - 2];
		const int32_t d3 = d[k < 3 ? p - 3 - back : p - 3], d4 = d[k < 4 ? p - 4 - back : p - 4];
		const int32_t e1 = d0 - d1, e2 = d0 - 2 * d1 + d2, e3 = d0 - 3 * d1 + 3 * d2 - d3, e4 = d0 - 4 * d1 + 6 * d2 - 4 * d3 + d4;
		te[0] += sign * abs_u32(d0);
		te[1] += sign * abs_u32(e1);
		te[2] += sign * abs_u32(e2);
		te[3] += sign * abs_u32(e3);
		te[4] += sign * abs_u32(e4);
	};
	int end = 2 * q;  // where the lane before lane j stops summing: lane 1 starts at od_1 = q, right behind lane 0
	for(int j = 2; j <= 4; j++) {
		const int od = j < 4 ? (j * n) >> 2 : n;
		for(int p = end; p < od; p++) terms(p, kMaxFixedOrder, 0, ~0ull);  // between lanes j-1 and j, or behind lane 3
		if(j == 4) break;
		const int back = od - j * q;
#pragma unroll 1
		for(int k = 0; k < 4 && k < q && back; k++) {
			terms(od + k, kMaxFixedOrder, 0, ~0ull);
			terms(od + k, k, back, 1ull);
		}
		end = od + q;
	}
}

// Partition order / Rice parameter search of one candidate (find_best_partition_order_ + set_partitioned_rice_,
// stream_encoder.c:4701-5075), run by one whole warp. sums[0 .. 2^max_po) holds the candidate's |residual| sums per partition
// at max_po and is overwritten; tmp holds at least 2^(max_po-1) entries. params_all receives order po's Rice parameters at
// offset (1 << po) - 1. Returns the Rice bits of the best order (entropy-coding header included) and that order in *best_po.
__device__ __forceinline__ uint32_t rice_search_warp(const EncK &P, int bs, int order, int max_po, int min_po, unsigned long long *sums,
                                                     unsigned long long *tmp, uint8_t *params_all, int *best_po_out)
{
	const int lane = threadIdx.x & 31;
	uint32_t best_r = 0;
	int best_po = 0;
	unsigned long long *cur = sums, *nxt = tmp;
	for(int po = max_po; po >= min_po; po--) {
		const int nparts = 1 << po;
		const uint32_t pbase = (uint32_t)(bs >> po);
		const uint32_t div_base = 0x40000u / pbase;
		unsigned long long local = 0;
		for(int p = lane; p < nparts; p += 32) {
			uint32_t psamp = pbase, div = div_base;
			if(p == 0) { psamp -= (uint32_t)order; div = 0x40000u / psamp; }
			const unsigned long long mean = cur[p];
			uint32_t k;
			if(mean < 2 || (((mean - 1) * div) >> 18) == 0) k = 0;
			else k = ilog2_u64(((mean - 1) * div) >> 18) + 1;
			if(k >= (uint32_t)P.rice_limit) k = (uint32_t)P.rice_limit - 1;
			params_all[(1 << po) - 1 + p] = (uint8_t)k;
			local += count_rice_bits(k, psamp, mean);
		}
		unsigned long long total = warp_sum_u64(local) + (kEntropyTypeLen + kRiceOrderLen);
		const uint32_t bits = (uint32_t)(total < 0xffffffffull ? total : 0xffffffffull);
		if(best_r == 0 || bits < best_r) { best_r = bits; best_po = po; }
		if(po > min_po) {
			for(int j = lane; j < nparts / 2; j += 32) nxt[j] = cur[2 * j] + cur[2 * j + 1];
			unsigned long long *t = cur; cur = nxt; nxt = t;
			__syncwarp();
		}
	}
	*best_po_out = best_po;
	return best_r;
}

// block-wide exclusive scan for 256 threads; returns exclusive prefix, *total = sum
__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t *s_warp /*[9]*/, uint32_t *total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t inc = v;
#pragma unroll
	for(int o = 1; o < 32; o <<= 1) {
		const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
		if(lane >= o) inc += t;
	}
	if(lane == 31) s_warp[warp] = inc;
	__syncthreads();
	if(warp == 0) {
		uint32_t w = (lane < 8) ? s_warp[lane] : 0;
		uint32_t winc = w;
#pragma unroll
		for(int o = 1; o < 8; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
			if(lane >= o) winc += t;
		}
		if(lane < 8) s_warp[lane] = winc - w;
		if(lane == 7) s_warp[8] = winc;
	}
	__syncthreads();
	const uint32_t res = s_warp[warp] + inc - v;
	*total = s_warp[8];
	__syncthreads();
	return res;
}

// channel assignment of a block from its plans (stream_encoder.c:3937-3972): 0 independent, 1 left/side, 2 side/right, 3 mid/side
__device__ __forceinline__ int channel_assignment(const EncK &P, const SubframePlan *bp, int flags)
{
	int ca = 0;
	if(P.channels == 2 && P.do_ms) {
		if(P.loose_ms) ca = (flags & 2) ? 3 : 0;
		else {
			const uint32_t b0 = bp[0].est_bits + bp[1].est_bits, b1 = bp[0].est_bits + bp[3].est_bits;
			const uint32_t b2 = bp[1].est_bits + bp[3].est_bits, b3 = bp[2].est_bits + bp[3].est_bits;
			uint32_t mn = b0;
			if(b1 < mn) { mn = b1; ca = 1; }
			if(b2 < mn) { mn = b2; ca = 2; }
			if(b3 < mn) { mn = b3; ca = 3; }
		}
	}
	return ca;
}

// the signal coded as channel c of a frame with assignment ca
__device__ __forceinline__ int subframe_signal(const EncK &P, int ca, int c)
{
	if(P.channels != 2) return c;
	if(c == 0) return (ca == 0 || ca == 1) ? 0 : (ca == 2 ? 3 : 2);
	return (ca == 0 || ca == 2) ? 1 : 3;
}

// frame number of block blk of a launch (stream_encoder.c:3772: each file is its own stream, numbered from 0)
__device__ __forceinline__ uint32_t frame_number_of(const EncK &P, int blk)
{
	const uint32_t gblk = P.blk0 + (uint32_t)blk;
	if(P.frame_no) return P.frame_no[gblk];
	return P.first_frame + (P.file_blocks ? gblk % (uint32_t)P.file_blocks : gblk);
}

// one thread writes the frame header and its CRC-8 at bit 0 of the zeroed word buffer `words`
__device__ __forceinline__ void put_frame_header(const EncK &P, uint32_t *words, int bs, uint32_t frame_number, int ca, const FrameHdr &H)
{
	const uint32_t cac = ca_code(ca, P.channels), bpsc = bps_code(P.bps), nb = (H.bits >> 3) - 1;  // nb: bytes in front of the CRC-8
	uint32_t crc = 0, w = 0;
	for(uint32_t b = 0; b <= nb; b++) {
		const uint32_t byte = b < nb ? frame_header_byte(H, bs, P.sample_rate, frame_number, cac, bpsc, (int)b) : crc;
		crc = crc8_byte(crc, byte);
		w |= byte << (24 - 8 * (b & 3));
		if((b & 3) == 3 || b == nb) { words[b >> 2] = w; w = 0; }
	}
}

// bits of a subframe header + warm-up + predictor description (everything in front of the residual)
__device__ __forceinline__ uint32_t subframe_header_bits(const SubframePlan *pl)
{
	uint32_t b = kSubframeHeaderBits + (uint32_t)pl->wasted;
	if(pl->type == SF_CONSTANT) b += (uint32_t)pl->bps;
	else if(pl->type == SF_FIXED || pl->type == SF_LPC) {
		b += (uint32_t)pl->order * (uint32_t)pl->bps + kEntropyTypeLen + kRiceOrderLen;
		if(pl->type == SF_LPC) b += kQlpPrecisionLen + kQlpShiftLen + (uint32_t)pl->order * (uint32_t)pl->precision;
	}
	return b;
}

// one thread writes the subframe header + warm-up + predictor (stream_encoder_framing.c:393-520) at bit `bitpos` of `words`;
// g: the signal (warm-up samples / constant value)
__device__ __forceinline__ void put_subframe_header(uint32_t *words, uint32_t bitpos, const SubframePlan *pl, const int32_t *g)
{
	const int type = pl->type, order = pl->order, wasted = pl->wasted, sbps = pl->bps;
	BitPut bw;
	bw.init(words, bitpos);
	uint32_t tb;
	switch(type) {
		case SF_CONSTANT: tb = 0x00; break;
		case SF_VERBATIM: tb = 0x02; break;
		case SF_FIXED: tb = 0x10 | ((uint32_t)order << 1); break;
		default: tb = 0x40 | ((uint32_t)(order - 1) << 1); break;
	}
	bw.put(tb | (wasted ? 1u : 0u), 8);
	if(wasted) { bw.skip((uint32_t)wasted - 1); bw.put(1, 1); }
	if(type == SF_CONSTANT) bw.put(mask_bits(g[0], (uint32_t)sbps), (uint32_t)sbps);
	else if(type == SF_FIXED || type == SF_LPC) {
		for(int i = 0; i < order; i++) bw.put(mask_bits(g[i], (uint32_t)sbps), (uint32_t)sbps);
		if(type == SF_LPC) {
			bw.put((uint32_t)pl->precision - 1, kQlpPrecisionLen);
			bw.put(mask_bits(pl->shift, kQlpShiftLen), kQlpShiftLen);
			for(int i = 0; i < order; i++) bw.put(mask_bits(pl->qlp[i], (uint32_t)pl->precision), (uint32_t)pl->precision);
		}
		bw.put((uint32_t)pl->method, kEntropyTypeLen);
		bw.put((uint32_t)pl->porder, kRiceOrderLen);
	}
	bw.finish();
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
