// glibc_tanh.cuh -- fb_tanh: the host libm's tanh() restated bit for bit, for the hard limiter of
// FLAC__replaygain_synthesis__apply_gain (replaygain_synthesis.c:374-380), which the flac tool runs on the host.
//
// glibc 2.39 on x86-64 builds tanh from the generic sysdeps/ieee754/dbl-64/s_tanh.c without FMA, and its call to expm1 goes
// through an ifunc that picks `__expm1_fma` (s_expm1.c built with -mfma -mavx2) on hosts with FMA and AVX2. CUDA's tanh is not
// that function, so this is the two routines transcribed from the binary's disassembly: the fused operations are explicit fb_fma
// calls exactly where the binary has vfmadd / vfmsub / vfnmadd, every other operation is a separately rounded double operation
// (the library is compiled with -fmad=false and the host side with -ffp-contract=off). Constants are the binary's.
// tests/test_gpu_decode_replaygain.py compares it with the host's tanh() bit for bit.
#pragma once

#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define FB_HD __host__ __device__ __forceinline__
#else
#define FB_HD inline
#endif
#ifndef __CUDA_ARCH__
#include <cmath>
#endif

namespace fb200 {

FB_HD double fb_fma(double a, double b, double c)
{
#ifdef __CUDA_ARCH__
	return __fma_rn(a, b, c);
#else
	return std::fma(a, b, c);
#endif
}

FB_HD uint64_t fb_bits(double x)
{
	uint64_t u;
	memcpy(&u, &x, 8);
	return u;
}

FB_HD double fb_from_bits(uint64_t u)
{
	double x;
	memcpy(&x, &u, 8);
	return x;
}

FB_HD double fb_set_high(double x, uint32_t hi) { return fb_from_bits((uint64_t)hi << 32 | (fb_bits(x) & 0xffffffffull)); }

// __expm1_fma for the arguments tanh gives it (finite, |x| < 44); the overflow and huge-negative branches are kept as written.
FB_HD double fb_expm1(double x)
{
	const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10, invln2 = 1.44269504088896338700e+00;
	const double Q1 = -3.33333333333331316428e-02, Q2 = 1.58730158725481460165e-03, Q3 = -7.93650757867487942473e-05,
	             Q4 = 4.00821782732936239552e-06, Q5 = -2.01099218183624371326e-07;
	const uint32_t hxa = (uint32_t)(fb_bits(x) >> 32);
	const bool neg = (hxa & 0x80000000u) != 0;
	const uint32_t hx = hxa & 0x7fffffffu;
	if(hx >= 0x4043687Au) {  // |x| >= 56 ln2
		if(hx >= 0x40862E42u) {
			if(hx >= 0x7ff00000u) return ((hx & 0xfffffu) | (uint32_t)fb_bits(x)) ? x + x : (neg ? -1.0 : x);
			if(x > 7.09782712893383973096e+02) return 1.0e+300 * 1.0e+300;
		}
		if(neg) return 1.0e-300 - 1.0;
	}
	double hi, lo, c = 0.0;
	int k;
	if(hx > 0x3fd62e42u) {  // |x| > 0.5 ln2
		if(hx < 0x3FF0A2B2u) {  // and < 1.5 ln2
			if(!neg) { hi = x - ln2_hi; lo = ln2_lo; k = 1; }
			else { hi = x + ln2_hi; lo = -ln2_lo; k = -1; }
		}
		else {
			k = (int)(invln2 * x + (neg ? -0.5 : 0.5));
			const double t = (double)k;
			hi = fb_fma(-t, ln2_hi, x);
			lo = t * ln2_lo;
		}
		const double xr = hi - lo;
		c = (hi - xr) - lo;
		x = xr;
	}
	else if(hx < 0x3c900000u) {  // |x| < 2^-54
		const double t = 1.0e+300 + x;
		return x - (t - (1.0e+300 + x));
	}
	else k = 0;
	const double hfx = x * 0.5;
	const double hxs = x * hfx;
	const double R2 = fb_fma(hxs, Q3, Q2);
	const double R3 = fb_fma(hxs, Q5, Q4);
	double h2 = hxs * hxs;
	const double R1 = fb_fma(hxs, Q1, 1.0);
	const double h4 = h2 * h2;
	h2 = fb_fma(h2, R2, R1);
	const double r1 = fb_fma(h4, R3, h2);
	const double t = fb_fma(-r1, hfx, 3.0);
	double e = (r1 - t) / fb_fma(-x, t, 6.0);
	e = e * hxs;
	if(k == 0) return x - fb_fma(e, x, -hxs);
	e = fb_fma(e - c, x, -c);
	e = e - hxs;
	if(k == -1) return fb_fma(0.5, x - e, -0.5);
	if(k == 1) {
		if(x < -0.25) return (e - (x + 0.5)) * -2.0;
		return fb_fma(x - e, 2.0, 1.0);
	}
	if(k <= -2 || k > 56) {
		double y = 1.0 - (e - x);
		y = fb_set_high(y, (uint32_t)(fb_bits(y) >> 32) + ((uint32_t)k << 20));
		return y - 1.0;
	}
	double y;
	if(k < 20) {
		const double t1 = fb_from_bits((uint64_t)(0x3ff00000u - (0x200000u >> k)) << 32);  // 1 - 2^-k
		y = t1 - (e - x);
	}
	else {
		const double t2 = fb_from_bits((uint64_t)((uint32_t)(0x3ff - k) << 20) << 32);  // 2^-k
		y = x - (e + t2);
		y = y + 1.0;
	}
	return fb_set_high(y, (uint32_t)(fb_bits(y) >> 32) + ((uint32_t)k << 20));
}

// s_tanh.c
FB_HD double fb_tanh(double x)
{
	const uint64_t u = fb_bits(x);
	const uint32_t jx = (uint32_t)(u >> 32), ix = jx & 0x7fffffffu, lx = (uint32_t)u;
	if(ix >= 0x7ff00000u) return (jx & 0x80000000u) ? 1.0 / x - 1.0 : 1.0 / x + 1.0;
	double z;
	if(ix < 0x40360000u) {  // |x| < 22
		if((ix | lx) == 0) return x;
		if(ix < 0x3c800000u) return (1.0 + x) * x;  // |x| < 2^-55
		const double ax = fb_from_bits(u & 0x7fffffffffffffffull);
		if(ix >= 0x3ff00000u) {  // |x| >= 1
			const double t = fb_expm1(ax + ax);
			z = 1.0 - 2.0 / (t + 2.0);
		}
		else {
			const double t = fb_expm1(ax * -2.0);
			z = -t / (t + 2.0);
		}
	}
	else z = 1.0 - 1.0e-300;
	return (jx & 0x80000000u) ? -z : z;
}

}  // namespace fb200
