// encode_kernels.cuh -- sm_90a kernels of the FLAC block encoder.
//
// Pipeline for a launch of N equal-sized blocks (frames are independent: SURVEY.md §0.1):
//   k_prep    : de-interleave, mid/side, wasted bits            (stream_encoder.c:3777-3867)
//   k_autoc   : windowed autocorrelation, one FP64 chain/thread  (lpc.c:68-174)
//   k_lpc     : Levinson-Durbin, order guess, quantisation       (lpc.c:176-314, 1580-1630)
//   k_search  : fixed scan + candidate residuals + Rice search   (stream_encoder.c:4045-4290, 4701-5075; fixed.c:222-290)
//   k_emit    : channel assignment, header, residual + Rice bit packing, CRC (stream_encoder.c:3934-4043,
//               stream_encoder_framing.c:245-594, bitwriter.c:575-706, crc.c)
//   k_scan / k_gather : frame offsets and contiguous stream.
//
// Floating point is evaluated in the reference's SOURCE order (no reassociation, no FMA
// contraction: compile with -fmad=false); everything after quantisation is integer.
#pragma once

#include "device_common.cuh"

namespace fb200 {

__global__ void k_debug_log(const double *__restrict__ x, double *__restrict__ y, int n)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) y[i] = fb_log(x[i]);
}

// ================================================================ k_unpack
// Packed little-endian signed PCM (2 or 3 bytes per sample, interleaved -- what a WAV/AIFF reader holds before the
// reference's client widens it to int32, src/flac/encode.c:2352 format_input) -> the interleaved int32 layout of
// FLAC__stream_encoder_process_interleaved. The only format-aware kernel: everything downstream sees int32.
// Samples outside the stream's bits_per_sample set *err = 3 (the reference's process() range check,
// stream_encoder.c:2543-2548).
template <int BYTES>
__global__ void __launch_bounds__(256) k_unpack(const uint8_t *__restrict__ packed, int32_t *__restrict__ pcm, unsigned long long n, int bps, int *__restrict__ err)
{
	// one thread = 4 consecutive samples: 8 (BYTES 2) or 12 (BYTES 3) input bytes -> one 16-byte store
	const unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
	const unsigned long long i0 = q * 4;
	if(i0 >= n) return;
	int v[4];
	const uint8_t *src = packed + i0 * BYTES;
	const bool full = i0 + 4 <= n;
	if(full && (((uintptr_t)src) & 3) == 0) {
		const uint32_t *w = reinterpret_cast<const uint32_t *>(src);
		if(BYTES == 2) {
			const uint32_t a = __ldg(w), b = __ldg(w + 1);
			v[0] = (int)(short)(a & 0xffffu); v[1] = (int)a >> 16; v[2] = (int)(short)(b & 0xffffu); v[3] = (int)b >> 16;
		}
		else {
			const uint32_t a = __ldg(w), b = __ldg(w + 1), c = __ldg(w + 2);
			v[0] = (int)(a << 8) >> 8;
			v[1] = (int)(((a >> 24) | (b << 8)) << 8) >> 8;
			v[2] = (int)(((b >> 16) | (c << 16)) << 8) >> 8;
			v[3] = (int)c >> 8;
		}
	}
	else {
#pragma unroll
		for(int e = 0; e < 4; e++) {
			v[e] = 0;
			if(i0 + e < n) {
				const uint8_t *p = src + e * BYTES;
				uint32_t u = (uint32_t)p[0] | ((uint32_t)p[1] << 8);
				if(BYTES == 3) u |= (uint32_t)p[2] << 16;
				v[e] = (int)(u << (32 - 8 * BYTES)) >> (32 - 8 * BYTES);
			}
		}
	}
	bool bad = false;
#pragma unroll
	for(int e = 0; e < 4; e++) {
		const int t = v[e] >> (bps - 1);
		bad |= (t != 0 && t != -1);
	}
	if(bad && bps < 8 * BYTES) atomicExch(err, 3);
	if(full) *reinterpret_cast<int4 *>(pcm + i0) = make_int4(v[0], v[1], v[2], v[3]);
	else
		for(int e = 0; e < 4 && i0 + e < n; e++) pcm[i0 + e] = v[e];
}

// ================================================================ k_prep
// One CTA per block. Signals are stored planar as sig[(blk*nsig + s)*bs_stride + i]:
// s < channels: the channel; s == channels: mid; s == channels+1: side. Wasted bits are
// shifted out here (get_wasted_bits_, stream_encoder.c:5077-5099), *after* mid/side were
// formed from the unshifted channels (:3823-3867). flags: bit0 do_independent, bit1 do_mid_side.
// WRITE_SIG = false is k_meta: wasted bits, subframe bps and the loose mid-side decision only -- the fast kernels
// (k_autoc4 / k_search5 / k_emit3) read the caller's interleaved PCM themselves and never need the planar copy.
template <bool WRITE_SIG>
__global__ void __launch_bounds__(256) k_prep(EncK P, const int32_t *__restrict__ pcm, int32_t *__restrict__ sig,
                                             SigMeta *__restrict__ meta, int *__restrict__ blkflags)
{
	const int blk = blockIdx.x, tid = threadIdx.x, ch = P.channels, bs = P.bs;
	const int32_t *src = pcm + (size_t)blk * bs * ch;
	__shared__ uint32_t s_or[FB200_MAX_CHANNELS + 2];
	__shared__ unsigned long long s_sum[2];
	if(tid < FB200_MAX_CHANNELS + 2) s_or[tid] = 0;
	if(tid < 2) s_sum[tid] = 0;
	__syncthreads();

	const bool stereo_ms = (ch == 2 && P.do_ms);
	uint32_t orv[FB200_MAX_CHANNELS + 2];
#pragma unroll
	for(int c = 0; c < FB200_MAX_CHANNELS + 2; c++) orv[c] = 0;
	unsigned long long sumLR = 0, sumMS = 0;

	if(stereo_ms) {
		const int2 *s2 = reinterpret_cast<const int2 *>(src);
		for(int i = tid; i < bs; i += blockDim.x) {
			const int2 v = s2[i];
			orv[0] |= (uint32_t)v.x;
			orv[1] |= (uint32_t)v.y;
			orv[2] |= (uint32_t)((v.x + v.y) >> 1);
			orv[3] |= (uint32_t)(v.x - v.y);
			if(P.loose_ms && i >= 1) {
				// loose mid-side heuristic (stream_encoder.c:3779-3807), bps < 25
				const int2 p = s2[i - 1];
				const int32_t pl = v.x - p.x, pr = v.y - p.y;
				sumLR += (unsigned long long)(abs(pl) + abs(pr));
				sumMS += (unsigned long long)(abs((pl + pr) >> 1) + abs(pl - pr));
			}
		}
	}
	else {
		for(int i = tid; i < bs; i += blockDim.x)
			for(int c = 0; c < ch; c++) orv[c] |= (uint32_t)src[(size_t)i * ch + c];
	}
	const int nsig = P.nsig;
	for(int s = 0; s < nsig; s++) {
		const uint32_t o = warp_or(orv[s]);
		if((tid & 31) == 0 && o) atomicOr(&s_or[s], o);
	}
	if(P.loose_ms) {
		sumLR = warp_sum_u64(sumLR);
		sumMS = warp_sum_u64(sumMS);
		if((tid & 31) == 0) { atomicAdd(&s_sum[0], sumLR); atomicAdd(&s_sum[1], sumMS); }
	}
	__syncthreads();

	int do_indep = 1, do_ms = 0;
	if(stereo_ms) {
		if(P.loose_ms) {
			if(s_sum[0] < s_sum[1]) { do_indep = 1; do_ms = 0; }
			else { do_indep = 0; do_ms = 1; }
		}
		else do_ms = 1;
	}
	int wasted[FB200_MAX_CHANNELS + 2];
	for(int s = 0; s < nsig; s++) {
		const uint32_t o = s_or[s];
		int w = o ? (__ffs((int)o) - 1) : 0;
		if(w > P.bps) w = P.bps;
		wasted[s] = w;
	}
	if(tid < nsig) {
		const bool active = (tid < ch) ? (do_indep != 0) : (do_ms != 0);
		SigMeta m;
		m.wasted = wasted[tid];
		m.bps = active ? (P.bps - wasted[tid] + ((stereo_ms && tid == ch + 1) ? 1 : 0)) : 0;
		meta[(size_t)blk * nsig + tid] = m;
	}
	if(tid == 0) blkflags[blk] = do_indep | (do_ms << 1);
	if(!WRITE_SIG) return;

	int32_t *dst = sig + (size_t)blk * nsig * P.bs_stride;
	if(stereo_ms) {
		const int2 *s2 = reinterpret_cast<const int2 *>(src);
		for(int i = tid; i < bs; i += blockDim.x) {
			const int2 v = s2[i];
			dst[i] = v.x >> wasted[0];
			dst[P.bs_stride + i] = v.y >> wasted[1];
			dst[2 * P.bs_stride + i] = ((v.x + v.y) >> 1) >> wasted[2];
			dst[3 * P.bs_stride + i] = (v.x - v.y) >> wasted[3];
		}
	}
	else {
		for(int i = tid; i < bs; i += blockDim.x)
			for(int c = 0; c < ch; c++) dst[(size_t)c * P.bs_stride + i] = src[(size_t)i * ch + c] >> wasted[c];
	}
}

// ================================================================ k_autoc
// autoc[l] = sum over ascending i of d[i]*d[i-l], one accumulator per lag (the source order of
// deduplication/lpc_compute_autocorrelation_intrin.c:5-14 and lpc.c:145-156). The order of
// additions is fixed, so a chain cannot be split across lanes; instead one THREAD owns one
// (block, signal, section) chain and keeps all LAGS accumulators plus a LAGS-deep history in
// registers: LAGS independent DFMAs per sample hide the FP64 latency. float*float products
// are exact in double, so fma() == mul+add here.
__device__ __forceinline__ float section_sample(const EncK &P, const DevSection &S, const int32_t *__restrict__ x,
                                                const float *__restrict__ w, int i)
{
	// lpc.c:68-94 FLAC__lpc_window_data / _partial: out = (float)in * window (one float rounding each)
	if(!S.partial)
		return __fmul_rn((float)__ldg(x + i), __ldg(w + i));
	if(i < S.part_size)
		return __fmul_rn((float)__ldg(x + S.data_shift + i), __ldg(w + i));
	if(i < 2 * S.part_size)
		return __fmul_rn((float)__ldg(x + S.data_shift + i), __ldg(w + (P.bs - 2 * S.part_size + i)));
	return 0.0f;
}

template <int LAGS>
__global__ void __launch_bounds__(128) k_autoc(EncK P, const int32_t *__restrict__ sig, const SigMeta *__restrict__ meta,
                                              const float *__restrict__ windows, const DevSection *__restrict__ secs,
                                              double *__restrict__ autoc, int nitems)
{
	const int gid = blockIdx.x * blockDim.x + threadIdx.x;
	if(gid >= nitems * P.nsec) return;
	const int sec = gid / nitems, item = gid - sec * nitems;
	if(meta[item].bps == 0) return;
	const DevSection S = secs[sec];
	const int32_t *x = sig + (size_t)item * P.bs_stride;
	const float *w = windows + S.win_off;
	const int n = S.data_len;

	double acc[LAGS], h[LAGS];
#pragma unroll
	for(int l = 0; l < LAGS; l++) { acc[l] = 0.0; h[l] = 0.0; }

	for(int base = 0; base < n; base += LAGS) {
#pragma unroll
		for(int u = 0; u < LAGS; u++) {
			const int i = base + u;
			const float d = (i < n) ? section_sample(P, S, x, w, i) : 0.0f;
			const double dv = (double)d;
			const int su = (LAGS - u) % LAGS;  // slot of the newest sample; slot (su+l)%LAGS holds d[i-l]
			h[su] = dv;
#pragma unroll
			for(int l = 0; l < LAGS; l++)
				acc[l] = fma(dv, h[(su + l) % LAGS], acc[l]);
		}
	}
	double *out = autoc + ((size_t)sec * nitems + item) * P.lag_stride;
#pragma unroll
	for(int l = 0; l < LAGS; l++) out[l] = acc[l];
}

// ================================================================ k_lpc

// lpc.c:1580-1606 FLAC__lpc_compute_expected_bits_per_residual_sample_with_error_scale
__device__ __forceinline__ double expected_bits_scale(double lpc_error, double error_scale)
{
	if(lpc_error > 0.0) {
		const double bps = (0.5 * fb_log(error_scale * lpc_error)) / M_LN2;
		return bps >= 0.0 ? bps : 0.0;
	}
	else if(lpc_error < 0.0)
		return 1e32;
	return 0.0;
}

// lpc.c:176-218 FLAC__lpc_compute_lp_coefficients. Runs the recursion up to max_order (or until the error hits 0.0),
// records the error per order and, when want_order > 0, the float predictor coefficients of that order. Returns the
// effective max order. Every loop is unrolled to the template bound MO with the live range as a predicate, so the
// working arrays stay in registers (round 1's run-time indexed version kept 1 KB of them in local memory per thread
// and stalled on those loads). The arithmetic -- operations and their order -- is the reference's, statement by statement.
template <int MO>
__device__ __forceinline__ int levinson(const double (&ac)[MO + 1], int max_order, int want_order, double (&err_out)[MO], float (&coef_out)[MO])
{
	double lpc[MO];
#pragma unroll
	for(int j = 0; j < MO; j++) lpc[j] = 0.0;
	double err = ac[0];
	int eff = max_order;
	bool done = false;
#pragma unroll
	for(int i = 0; i < MO; i++) {
		if(i < max_order && !done) {
			double r = -ac[i + 1];
#pragma unroll
			for(int j = 0; j < MO; j++)
				if(j < i) r -= lpc[j] * ac[i - j];
			r /= err;
			lpc[i] = r;
#pragma unroll
			for(int j = 0; j < MO / 2; j++)
				if(j < (i >> 1)) {
					const double tmp = lpc[j];
					lpc[j] += r * lpc[i - 1 - j];
					lpc[i - 1 - j] += r * tmp;
				}
			if(i & 1) lpc[i >> 1] += lpc[i >> 1] * r;
			err *= (1.0 - r * r);
			err_out[i] = err;
			if(i + 1 == want_order) {
#pragma unroll
				for(int k = 0; k < MO; k++)
					if(k <= i) coef_out[k] = (float)(-lpc[k]);
			}
			if(err == 0.0) { eff = i + 1; done = true; }
		}
	}
	return eff;
}

// lpc.c:220-314 FLAC__lpc_quantize_coefficients
template <int MO>
__device__ __forceinline__ int quantize_coefficients(const float (&lp_coeff)[MO], int order, int precision, int (&qlp)[MO], int *shift_out)
{
	precision--;
	int qmax = 1 << precision;
	const int qmin = -qmax;
	qmax--;
	double cmax = 0.0;
#pragma unroll
	for(int i = 0; i < MO; i++)
		if(i < order) {
			const double d = fabs((double)lp_coeff[i]);
			if(d > cmax) cmax = d;
		}
	if(cmax <= 0.0) return 2;
	int shift;
	{
		const int max_shiftlimit = (1 << (kQlpShiftLen - 1)) - 1;
		const int min_shiftlimit = -max_shiftlimit - 1;
		int log2cmax;
		(void)frexp(cmax, &log2cmax);
		log2cmax--;
		shift = precision - log2cmax - 1;
		if(shift > max_shiftlimit) shift = max_shiftlimit;
		else if(shift < min_shiftlimit) return 1;
	}
	double error = 0.0;
	if(shift >= 0) {
		const float scale = (float)(1 << shift);
#pragma unroll
		for(int i = 0; i < MO; i++)
			if(i < order) {
				error += (double)__fmul_rn(lp_coeff[i], scale);
				long long q = llround(error);
				if(q > qmax) q = qmax;
				else if(q < qmin) q = qmin;
				error -= (double)q;
				qlp[i] = (int)q;
			}
	}
	else {
		const float scale = (float)(1 << (-shift));
#pragma unroll
		for(int i = 0; i < MO; i++)
			if(i < order) {
				error += (double)__fdiv_rn(lp_coeff[i], scale);
				long long q = llround(error);
				if(q > qmax) q = qmax;
				else if(q < qmin) q = qmin;
				error -= (double)q;
				qlp[i] = (int)q;
			}
		shift = 0;
	}
	*shift_out = shift;
	return 0;
}

// One thread per (block, signal, window candidate). Writes nslots/nwin candidate slots.
// autoc_unshifted: the autocorrelation was taken over the signal BEFORE its wasted bits were shifted out (k_autoc4 running
// concurrently with k_meta): autoc(x >> w) = autoc(x) * 2^-2w exactly, applied here.
template <int MO>
__global__ void __launch_bounds__(128) k_lpc(EncK P, const double *__restrict__ autoc, const DevCand *__restrict__ cands,
                                            SigMeta *__restrict__ meta, const uint32_t *__restrict__ sigor, CandDesc *__restrict__ out, int nitems,
                                            int autoc_unshifted)
{
	const int gid = blockIdx.x * blockDim.x + threadIdx.x;
	if(gid >= nitems * P.nwin) return;
	const int win = gid / nitems, item = gid - win * nitems;
	const int per_win = P.nslots / P.nwin;
	CandDesc *slots = out + ((size_t)item * P.nslots + (size_t)win * per_win);
	for(int s = 0; s < per_win; s++) slots[s].valid = 0;
	SigMeta M;
	if(sigor) {
		// the OR of the signal's samples came with the autocorrelation (k_autoc4): wasted bits and subframe bps as k_meta
		// derives them (get_wasted_bits_, stream_encoder.c:5077-5099; side channel one bit wider, :3865); every signal is active
		const uint32_t o = sigor[item];
		int w = o ? (__ffs((int)o) - 1) : 0;
		if(w > P.bps) w = P.bps;
		const int sidx = item % P.nsig;
		M.wasted = w;
		M.bps = P.bps - w + ((P.channels == 2 && P.nsig == 4 && sidx == 3) ? 1 : 0);
		if(win == 0) meta[item] = M;  // k_search5 reads it from here
	}
	else M = meta[item];
	const int sbps = M.bps;
	if(sbps == 0) return;

	const int max_order = P.max_order;
	const DevCand C = cands[win];
	double ac[MO + 1];
	{
		const double *a = autoc + ((size_t)C.sec * nitems + item) * P.lag_stride;
		// 2^-2w (1.0 when nothing is to undo): an exact scaling of every sum
		const double sc = autoc_unshifted ? __hiloint2double((1023 - 2 * M.wasted) << 20, 0) : 1.0;
		if(C.kind == 0) {
#pragma unroll
			for(int l = 0; l <= MO; l++) ac[l] = l <= max_order ? a[l] * sc : 0.0;
		}
		else {
			// punch-out = root - partial over max_order entries; entry [max_order] keeps the partial
			// window's value (stream_encoder.c:4339-4340, 4370-4371).
			const double *r = autoc + ((size_t)C.root * nitems + item) * P.lag_stride;
#pragma unroll
			for(int l = 0; l <= MO; l++) ac[l] = l < max_order ? r[l] * sc - a[l] * sc : (l == max_order ? a[l] * sc : 0.0);
		}
	}
	if(ac[0] == 0.0) return;

	double lpc_error[MO];
	float coef[MO];
#pragma unroll
	for(int i = 0; i < MO; i++) { lpc_error[i] = 0.0; coef[i] = 0.0f; }
	const int eff_max = levinson<MO>(ac, max_order, 0, lpc_error, coef);

	int lo, hi;
	if(P.exhaustive) { lo = 1; hi = eff_max; }
	else {
		// lpc.c:1608-1630 FLAC__lpc_compute_best_order
		const uint32_t total_samples = (uint32_t)P.bs;
		const uint32_t overhead = (uint32_t)(sbps + (P.prec_search ? (int)kMinQlpPrecision : P.qlp_precision));  // stream_encoder.c:4385-4389
		const double error_scale = 0.5 / (double)total_samples;
		int best_index = 0;
		double best_bits = (double)0xffffffffu;
#pragma unroll
		for(int indx = 0; indx < MO; indx++)
			if(indx < eff_max) {
				const uint32_t order = (uint32_t)indx + 1;
				const double bits = expected_bits_scale(lpc_error[indx], error_scale) * (double)(total_samples - order) + (double)(order * overhead);
				if(bits < best_bits) { best_index = indx; best_bits = bits; }
			}
		lo = hi = best_index + 1;
	}
	const int nprec = P.prec_search ? kQlpPrecisionSteps : 1;
	for(int order = lo; order <= hi; order++) {
		double err_o = 0.0;
#pragma unroll
		for(int i = 0; i < MO; i++)
			if(i == order - 1) err_o = lpc_error[i];
		// stream_encoder.c:4227-4229 "don't even try"
		const double lbps = expected_bits_scale(err_o, 0.5 / (double)(uint32_t)(P.bs - order));
		if(lbps >= (double)sbps) continue;
		// precisions tried for this order (:4230-4243): the configured one, or 5 .. 15 (<= 17-bit subframes: capped so that the
		// decoder's 32-bit arithmetic suffices)
		int minp = P.qlp_precision, maxp = P.qlp_precision;
		if(P.prec_search) {
			minp = (int)kMinQlpPrecision;
			maxp = (int)kMaxQlpPrecision;
			if(sbps <= 17) maxp = max(min(32 - sbps - (int)ilog2_u32((uint32_t)order), (int)kMaxQlpPrecision), minp);
		}
		double scratch_err[MO];
		(void)levinson<MO>(ac, order, order, scratch_err, coef);
		for(int prec_try = minp; prec_try <= maxp; prec_try++) {
		CandDesc &D = slots[(order - lo) * nprec + (prec_try - minp)];
		int precision = prec_try;
		if(sbps <= 17) precision = min(precision, 32 - sbps - (int)ilog2_u32((uint32_t)order));  // :4591-4595
		int q[MO], shift;
#pragma unroll
		for(int i = 0; i < MO; i++) q[i] = 0;
		if(quantize_coefficients<MO>(coef, order, precision, q, &shift) != 0) continue;
		// lpc.c:942-968
		uint32_t abs_sum = 0;
#pragma unroll
		for(int i = 0; i < MO; i++)
			if(i < order) abs_sum += (uint32_t)abs(q[i]);
		const uint64_t max_abs_sample = (uint64_t)1 << (sbps - 1);
		const uint64_t max_pred = max_abs_sample * abs_sum;
		const uint64_t max_pred_after = (uint64_t)(-1 * ((-1 * (int64_t)max_pred) >> shift));
		D.limit = silog2_i64((int64_t)(max_abs_sample + max_pred_after)) > 32;
		D.wide = (silog2_i64((int64_t)max_pred) > 32) || D.limit;  // the checked variant is 64-bit (lpc.c:786-884)
		D.order = order;
		D.precision = precision;
		D.shift = shift;
#pragma unroll
		for(int i = 0; i < FB200_MAX_LPC_ORDER; i++) D.qlp[i] = (i < MO && i < order) ? q[i < MO ? i : 0] : 0;
		D.valid = 1;
		}
	}
}

// ================================================================ k_minbr_flags
// limit_min_bitrate (stream_encoder.c:3874-3879): when every independent channel before the last chose a CONSTANT subframe,
// the last channel -- and the mid/side pair evaluated after it -- is searched with constant subframes disabled. The first
// search pass ran every signal with the stream's own settings; this marks the blocks whose last channel / mid / side are
// searched again (P.redo) with constants off.
__global__ void k_minbr_flags(EncK P, const SubframePlan *__restrict__ plans, const int *__restrict__ blkflags, int nb, int *__restrict__ flags)
{
	const int blk = blockIdx.x * blockDim.x + threadIdx.x;
	if(blk >= nb) return;
	bool all_const = blkflags ? (blkflags[blk] & 1) != 0 : true;  // only inside the independent-channel loop
	for(int c = 0; c + 1 < P.channels; c++) all_const = all_const && plans[(size_t)blk * P.nsig + c].type == SF_CONSTANT;
	flags[blk] = all_const ? 1 : 0;
}

// ================================================================ k_search
// One CTA (128 threads) per (block, signal). The signal sits in shared memory; every
// candidate predictor is run over it, |residual| goes to shared memory, partition sums are
// reduced per warp and warp 0 does the partition-order/Rice-parameter search.

struct SearchShared {
	unsigned long long sums[2][kMaxPartitions];
	unsigned long long te[5];
	uint8_t params_all[2 * kMaxPartitions];  // order po at offset (1<<po)-1
	int fail;
	int all_equal;
	uint32_t best_bits;
	// best plan so far
	int b_type, b_order, b_prec, b_shift, b_method, b_po, b_wide;
	int b_qlp[FB200_MAX_LPC_ORDER];
	uint8_t b_params[kMaxPartitions];
	// current candidate
	int c_qlp[FB200_MAX_LPC_ORDER];
};

// Evaluate one predictor on the block in shared memory and, if it beats the best-so-far
// (strict '<', stream_encoder.c:4191-4194, 4265-4269), record it. type: SF_FIXED or SF_LPC.
__device__ void evaluate_candidate(const EncK &P, SearchShared &S, const int32_t *__restrict__ x, uint32_t *__restrict__ absr,
                                   int type, int order, int precision, int shift, int wide, int limit, int sbps, int wasted)
{
	const int tid = threadIdx.x, bs = P.bs, nthr = blockDim.x;
	const int nres = bs - order;

	// --- residual magnitudes (fixed.c:470-530, lpc.c:321-938; int64 == every variant, see oracle)
	if(type == SF_FIXED) {
		for(int i = order + tid; i < bs; i += nthr) {
			int32_t r;
			switch(order) {
				case 0: r = x[i]; break;
				case 1: r = x[i] - x[i - 1]; break;
				case 2: r = x[i] - 2 * x[i - 1] + x[i - 2]; break;
				case 3: r = x[i] - 3 * x[i - 1] + 3 * x[i - 2] - x[i - 3]; break;
				default: r = x[i] - 4 * x[i - 1] + 6 * x[i - 2] - 4 * x[i - 3] + x[i - 4]; break;
			}
			absr[i - order] = abs_u32(r);
		}
	}
	else if(!wide) {
		for(int i = order + tid; i < bs; i += nthr) {
			int32_t sum = 0;
			for(int j = 0; j < order; j++) sum += S.c_qlp[j] * x[i - 1 - j];
			absr[i - order] = abs_u32(x[i] - (sum >> shift));
		}
	}
	else {
		bool bad = false;
		for(int i = order + tid; i < bs; i += nthr) {
			int64_t sum = 0;
			for(int j = 0; j < order; j++) sum += (int64_t)S.c_qlp[j] * (int64_t)x[i - 1 - j];
			const int64_t r = (int64_t)x[i] - (sum >> shift);
			if(limit && (r <= (int64_t)INT32_MIN || r > (int64_t)INT32_MAX)) bad = true;  // lpc.c:868-884
			absr[i - order] = abs_u32((int32_t)r);
		}
		if(bad) S.fail = 1;
	}
	__syncthreads();
	if(S.fail) {  // candidate rejected (evaluate_lpc_subframe_ returns 0, stream_encoder.c:4601-4609)
		__syncthreads();
		if(tid == 0) S.fail = 0;
		__syncthreads();
		return;
	}

	// --- partition sums at the largest usable order (stream_encoder.c:4797-4835)
	int max_po = P.max_po;
	while(max_po > 0 && (bs >> max_po) <= order) max_po--;  // format.c:550-562
	const int min_po = min(P.min_po, max_po);
	{
		const int psize = bs >> max_po, nparts = 1 << max_po;
		const bool narrow = (uint32_t)(sbps + (int)kMaxExtraResidualBps) < 32u - ilog2_u32((uint32_t)psize);
		const int warp = tid >> 5, lane = tid & 31, nwarps = nthr >> 5;
		for(int p = warp; p < nparts; p += nwarps) {
			const int start = (p == 0) ? 0 : p * psize - order;
			const int end = (p + 1) * psize - order;
			unsigned long long s = 0;
			for(int j = start + lane; j < end; j += 32) s += absr[j];
			s = warp_sum_u64(s);
			if(lane == 0) S.sums[0][p] = narrow ? (unsigned long long)(uint32_t)s : s;
		}
	}
	__syncthreads();

	// --- warp 0: partition order search (find_best_partition_order_ + set_partitioned_rice_, :4701-5075)
	if(tid < 32) {
		const int lane = tid;
		uint32_t best_r = 0;
		int best_po = 0, cur = 0;
		for(int po = max_po; po >= min_po; po--) {
			const int nparts = 1 << po;
			const uint32_t pbase = (uint32_t)(bs >> po);
			const uint32_t div_base = 0x40000u / pbase;
			unsigned long long local = 0;
			for(int p = lane; p < nparts; p += 32) {
				uint32_t psamp = pbase, div = div_base;
				if(p == 0) { psamp -= (uint32_t)order; div = 0x40000u / psamp; }
				const unsigned long long mean = S.sums[cur][p];
				uint32_t k;
				if(mean < 2 || (((mean - 1) * div) >> 18) == 0) k = 0;
				else k = ilog2_u64(((mean - 1) * div) >> 18) + 1;
				if(k >= (uint32_t)P.rice_limit) k = (uint32_t)P.rice_limit - 1;
				S.params_all[(1 << po) - 1 + p] = (uint8_t)k;
				local += count_rice_bits(k, psamp, mean);
			}
			unsigned long long total = warp_sum_u64(local) + (kEntropyTypeLen + kRiceOrderLen);
			const uint32_t bits = (uint32_t)(total < 0xffffffffull ? total : 0xffffffffull);
			if(best_r == 0 || bits < best_r) { best_r = bits; best_po = po; }
			if(po > min_po) {
				for(int j = lane; j < nparts / 2; j += 32) S.sums[cur ^ 1][j] = S.sums[cur][2 * j] + S.sums[cur][2 * j + 1];
				cur ^= 1;
				__syncwarp();
			}
		}
		// estimate (evaluate_fixed_subframe_ :4550-4554, evaluate_lpc_subframe_ :4655-4659)
		uint32_t estimate = kSubframeHeaderBits + (uint32_t)wasted;
		if(type == SF_FIXED) estimate += (uint32_t)order * (uint32_t)sbps;
		else estimate += kQlpPrecisionLen + kQlpShiftLen + (uint32_t)order * (uint32_t)(precision + sbps);
		if(best_r < 0xffffffffu - estimate) estimate += best_r;
		else estimate = 0xffffffffu;
		const bool better = (type == SF_LPC ? estimate > 0 : true) && estimate < S.best_bits;
		if(better) {
			const int nparts = 1 << best_po;
			uint32_t any15 = 0;
			for(int p = lane; p < nparts; p += 32) {
				const uint8_t k = S.params_all[(1 << best_po) - 1 + p];
				S.b_params[p] = k;
				any15 |= (k >= kRiceEscape) ? 1u : 0u;
			}
			any15 = warp_or(any15);
			if(lane < FB200_MAX_LPC_ORDER) S.b_qlp[lane] = (type == SF_LPC && lane < order) ? S.c_qlp[lane] : 0;
			if(lane == 0) {
				S.best_bits = estimate;
				S.b_type = type; S.b_order = order; S.b_prec = precision; S.b_shift = shift;
				S.b_method = any15 ? 1 : 0;  // RICE2 when a parameter needs 5 bits (:4786-4791)
				S.b_po = best_po; S.b_wide = wide;
			}
		}
	}
	__syncthreads();
}

__global__ void __launch_bounds__(128) k_search(EncK P, const int32_t *__restrict__ sig, const SigMeta *__restrict__ meta,
                                               const CandDesc *__restrict__ cdesc, SubframePlan *__restrict__ plans)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	__shared__ SearchShared S;
	const int item = blockIdx.x, tid = threadIdx.x, bs = P.bs, nthr = blockDim.x;
	if(P.redo) {
		const int blk = item / P.nsig;
		if(!P.redo[blk] || item - blk * P.nsig < P.channels - 1) return;
	}
	int32_t *x = reinterpret_cast<int32_t *>(smem_raw);
	uint32_t *absr = reinterpret_cast<uint32_t *>(x + P.bs_stride);

	const SigMeta M = meta[item];
	SubframePlan *plan = plans + item;
	if(M.bps == 0) {
		if(tid == 0) { plan->type = -1; plan->est_bits = 0xffffffffu; }
		return;
	}
	const int sbps = M.bps, wasted = M.wasted;
	const int32_t *g = sig + (size_t)item * P.bs_stride;
	for(int i = tid; i < bs; i += nthr) x[i] = g[i];
	if(tid == 0) {
		S.fail = 0; S.all_equal = 1;
		// verbatim baseline (evaluate_verbatim_subframe_, :4669-4699; :4082-4086)
		S.b_type = SF_VERBATIM; S.b_order = 0; S.b_prec = 0; S.b_shift = 0; S.b_method = 0; S.b_po = 0; S.b_wide = 0;
		if(P.dis_verb && bs >= (int)kMaxFixedOrder) S.best_bits = 0xffffffffu;
		else S.best_bits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)bs * (uint32_t)sbps;
	}
	if(tid < 5) S.te[tid] = 0;
	__syncthreads();

	if(bs > (int)kMaxFixedOrder) {
		// fixed.c:222-290: abs sums of the 0..4th differences over samples 4..bs-1
		unsigned long long te[5] = {0, 0, 0, 0, 0};
		for(int i = (int)kMaxFixedOrder + tid; i < bs; i += nthr) {
			const int64_t d0 = x[i], d1 = x[i - 1], d2 = x[i - 2], d3 = x[i - 3], d4 = x[i - 4];
			const int64_t e1 = d0 - d1, e2 = d0 - 2 * d1 + d2, e3 = d0 - 3 * d1 + 3 * d2 - d3, e4 = d0 - 4 * d1 + 6 * d2 - 4 * d3 + d4;
			te[0] += (unsigned long long)(d0 < 0 ? -d0 : d0);
			te[1] += (unsigned long long)(e1 < 0 ? -e1 : e1);
			te[2] += (unsigned long long)(e2 < 0 ? -e2 : e2);
			te[3] += (unsigned long long)(e3 < 0 ? -e3 : e3);
			te[4] += (unsigned long long)(e4 < 0 ? -e4 : e4);
		}
#pragma unroll
		for(int k = 0; k < 5; k++) {
			te[k] = warp_sum_u64(te[k]);
			if((tid & 31) == 0) atomicAdd(&S.te[k], te[k]);
		}
		__syncthreads();
		unsigned long long t0 = S.te[0], t1 = S.te[1], t2 = S.te[2], t3 = S.te[3], t4 = S.te[4];
		int guess;
		{
			const unsigned long long m34 = t3 < t4 ? t3 : t4, m234 = t2 < m34 ? t2 : m34, m1234 = t1 < m234 ? t1 : m234;
			if(t0 <= m1234) guess = 0;
			else if(t1 <= m234) guess = 1;
			else if(t2 <= m34) guess = 2;
			else if(t3 <= t4) guess = 3;
			else guess = 4;
		}
		float rbps[5];
		{
			const double n = (double)(uint32_t)(bs - (int)kMaxFixedOrder);
			const unsigned long long tt[5] = {t0, t1, t2, t3, t4};
#pragma unroll
			for(int k = 0; k < 5; k++)
				rbps[k] = (float)((tt[k] > 0) ? fb_log(M_LN2 * (double)tt[k] / n) / M_LN2 : 0.0);
		}
		bool is_constant = false;
		if(!P.dis_const && rbps[1] == 0.0f) {
			// stream_encoder.c:4111-4140
			uint32_t eq = 1;
			const int32_t x0 = x[0];
			for(int i = 1 + tid; i < bs; i += nthr) eq &= (x[i] == x0) ? 1u : 0u;
			eq = warp_and(eq);
			if((tid & 31) == 0 && !eq) S.all_equal = 0;
			__syncthreads();
			is_constant = S.all_equal != 0;
		}
		if(is_constant) {
			if(tid == 0) {
				const uint32_t cbits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)sbps;  // :4466-4487
				if(cbits < S.best_bits) { S.best_bits = cbits; S.b_type = SF_CONSTANT; }
			}
			__syncthreads();
		}
		else {
			if(!P.dis_fixed || (P.max_order == 0 && S.best_bits == 0xffffffffu)) {
				int lo, hi;
				if(P.exhaustive) { lo = 0; hi = (int)kMaxFixedOrder; }
				else lo = hi = guess;
				if(hi >= bs) hi = bs - 1;
				for(int fo = lo; fo <= hi; fo++) {
					if(rbps[fo] >= (float)sbps) continue;  // :4166
					evaluate_candidate(P, S, x, absr, SF_FIXED, fo, 0, 0, 0, 0, sbps, wasted);
				}
			}
			if(P.max_order > 0) {
				const CandDesc *cd = cdesc + (size_t)item * P.nslots;
				for(int c = 0; c < P.nslots; c++) {
					const CandDesc *D = cd + c;
					if(!D->valid) continue;
					if(tid < FB200_MAX_LPC_ORDER) S.c_qlp[tid] = D->qlp[tid];
					__syncthreads();
					evaluate_candidate(P, S, x, absr, SF_LPC, D->order, D->precision, D->shift, D->wide, D->limit, sbps, wasted);
				}
			}
		}
	}
	__syncthreads();
	if(S.best_bits == 0xffffffffu) {  // :4281-4284
		if(tid == 0) {
			S.b_type = SF_VERBATIM;
			S.best_bits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)bs * (uint32_t)sbps;
		}
		__syncthreads();
	}
	if(tid == 0) {
		plan->type = S.b_type; plan->order = S.b_order; plan->wasted = wasted; plan->bps = sbps;
		plan->precision = S.b_prec; plan->shift = S.b_shift; plan->method = S.b_method; plan->porder = S.b_po;
		plan->est_bits = S.best_bits; plan->wide = S.b_wide;
	}
	if(tid < FB200_MAX_LPC_ORDER) plan->qlp[tid] = S.b_qlp[tid];
	for(int p = tid; p < kMaxPartitions; p += nthr) plan->params[p] = S.b_params[p];
}

// ================================================================ k_emit
// One CTA (256 threads) per frame. MSB-first bit packing into a shared-memory word buffer:
// each thread owns a contiguous run of samples, a block-wide prefix sum of the run bit
// lengths gives every run its start bit, runs are packed independently (only the first and
// the last word of a run can be shared with a neighbour -> atomicOr), then CRC-16 is
// computed in parallel by chunk + GF(2) combine, and the frame is copied to its slot.

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

__global__ void __launch_bounds__(256) k_emit(EncK P, const int32_t *__restrict__ sig, const int *__restrict__ blkflags,
                                             const SubframePlan *__restrict__ plans, uint8_t *__restrict__ slots,
                                             uint32_t *__restrict__ frame_bytes, uint32_t *__restrict__ chan_assign_out)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int blk = blockIdx.x, tid = threadIdx.x, bs = P.bs, nthr = 256;
	const int xcap = skew(P.bs_stride) + 1;
	int32_t *x = reinterpret_cast<int32_t *>(smem_raw);
	int32_t *res = x + xcap;
	uint32_t *words = reinterpret_cast<uint32_t *>(res + xcap);
	__shared__ uint16_t s_crctab[256];
	__shared__ uint32_t s_warp[9];
	__shared__ uint32_t s_crc[256];
	__shared__ uint32_t s_mlev[8];
	__shared__ int s_ca;

	for(int i = tid; i < P.slot_words; i += nthr) words[i] = 0;
	{   // CRC-16 table entry (crc.c:78-342)
		uint32_t c = (uint32_t)tid << 8;
#pragma unroll
		for(int j = 0; j < 8; j++) c = (c & 0x8000u) ? ((c << 1) ^ 0x8005u) : (c << 1);
		s_crctab[tid] = (uint16_t)c;
	}
	const SubframePlan *bp = plans + (size_t)blk * P.nsig;
	if(tid == 0) {
		// channel assignment (stream_encoder.c:3937-3972)
		int ca = 0;
		const int flags = blkflags[blk];
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
		s_ca = ca;
	}
	__syncthreads();
	const int ca = s_ca;
	const uint32_t gblk = P.blk0 + (uint32_t)blk;
	const uint32_t frame_number = P.first_frame + (P.file_blocks ? gblk % (uint32_t)P.file_blocks : gblk);

	// ---- frame header (stream_encoder_framing.c:245-391), thread 0
	uint32_t bs_code, bs_hint = 0, sr_code, sr_hint = 0;
	switch(bs) {
		case 192: bs_code = 1; break; case 576: bs_code = 2; break; case 1152: bs_code = 3; break;
		case 2304: bs_code = 4; break; case 4608: bs_code = 5; break; case 256: bs_code = 8; break;
		case 512: bs_code = 9; break; case 1024: bs_code = 10; break; case 2048: bs_code = 11; break;
		case 4096: bs_code = 12; break; case 8192: bs_code = 13; break; case 16384: bs_code = 14; break;
		case 32768: bs_code = 15; break;
		default: bs_code = bs_hint = (bs <= 0x100) ? 6 : 7; break;
	}
	switch(P.sample_rate) {
		case 88200: sr_code = 1; break; case 176400: sr_code = 2; break; case 192000: sr_code = 3; break;
		case 8000: sr_code = 4; break; case 16000: sr_code = 5; break; case 22050: sr_code = 6; break;
		case 24000: sr_code = 7; break; case 32000: sr_code = 8; break; case 44100: sr_code = 9; break;
		case 48000: sr_code = 10; break; case 96000: sr_code = 11; break;
		default:
			if(P.sample_rate <= 255000 && P.sample_rate % 1000 == 0) sr_code = sr_hint = 12;
			else if(P.sample_rate <= 655350 && P.sample_rate % 10 == 0) sr_code = sr_hint = 14;
			else if(P.sample_rate <= 0xffff) sr_code = sr_hint = 13;
			else sr_code = 0;
			break;
	}
	uint32_t utf8_len;
	if(frame_number < 0x80) utf8_len = 1;
	else if(frame_number < 0x800) utf8_len = 2;
	else if(frame_number < 0x10000) utf8_len = 3;
	else if(frame_number < 0x200000) utf8_len = 4;
	else if(frame_number < 0x4000000) utf8_len = 5;
	else utf8_len = 6;
	const uint32_t header_bits = 32 + 8 * utf8_len + (bs_hint ? (bs_hint == 6 ? 8 : 16) : 0) + (sr_hint ? (sr_hint == 12 ? 8 : 16) : 0) + 8;

	if(tid == 0) {
		BitPut bw;
		bw.init(words, 0);
		uint32_t ca_code;
		switch(ca) { case 0: ca_code = (uint32_t)P.channels - 1; break; case 1: ca_code = 8; break; case 2: ca_code = 9; break; default: ca_code = 10; break; }
		uint32_t bps_code;
		switch(P.bps) { case 8: bps_code = 1; break; case 12: bps_code = 2; break; case 16: bps_code = 4; break; case 20: bps_code = 5; break; case 24: bps_code = 6; break; case 32: bps_code = 7; break; default: bps_code = 0; break; }
		bw.put(0x3ffe, 14); bw.put(0, 1); bw.put(0, 1);
		bw.put(bs_code, 4); bw.put(sr_code, 4); bw.put(ca_code, 4); bw.put(bps_code, 3); bw.put(0, 1);
		// UTF-8 style frame number (bitwriter.c:832-933)
		const uint32_t v = frame_number;
		switch(utf8_len) {
			case 1: bw.put(v, 8); break;
			case 2: bw.put(0xC0 | (v >> 6), 8); break;
			case 3: bw.put(0xE0 | (v >> 12), 8); break;
			case 4: bw.put(0xF0 | (v >> 18), 8); break;
			case 5: bw.put(0xF8 | (v >> 24), 8); break;
			default: bw.put(0xFC | (v >> 30), 8); break;
		}
		for(int k = (int)utf8_len - 2; k >= 0; k--) bw.put(0x80 | ((v >> (6 * k)) & 0x3F), 8);
		if(bs_hint) bw.put((uint32_t)bs - 1, bs_hint == 6 ? 8 : 16);
		if(sr_hint == 12) bw.put((uint32_t)P.sample_rate / 1000, 8);
		else if(sr_hint == 13) bw.put((uint32_t)P.sample_rate, 16);
		else if(sr_hint == 14) bw.put((uint32_t)P.sample_rate / 10, 16);
		bw.finish();
		// CRC-8, poly 0x07 (crc.c:39-76), over the header bytes written so far
		const uint32_t nb = (header_bits - 8) >> 3;
		uint32_t crc = 0;
		for(uint32_t b = 0; b < nb; b++) {
			crc ^= (words[b >> 2] >> (24 - 8 * (b & 3))) & 0xffu;
			for(int j = 0; j < 8; j++) crc = (crc & 0x80u) ? ((crc << 1) ^ 0x07u) & 0xffu : (crc << 1) & 0xffu;
		}
		bw.init(words, header_bits - 8);
		bw.put(crc, 8);
		bw.finish();
	}
	__syncthreads();

	uint32_t bitpos = header_bits;
	for(int c = 0; c < P.channels; c++) {
		int sidx = c;
		if(P.channels == 2) {
			if(c == 0) sidx = (ca == 0 || ca == 1) ? 0 : (ca == 2 ? 3 : 2);
			else sidx = (ca == 0 || ca == 2) ? 1 : 3;
		}
		const SubframePlan *pl = bp + sidx;
		const int type = pl->type, order = pl->order, wasted = pl->wasted, sbps = pl->bps;
		const int32_t *g = sig + ((size_t)blk * P.nsig + sidx) * P.bs_stride;
		const uint32_t hdr_bits = kSubframeHeaderBits + (uint32_t)wasted;  // wasted: unary w-1 zeros + 1

		if(tid == 0) {
			// subframe header + warm-up + predictor (stream_encoder_framing.c:393-520)
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
		bitpos += hdr_bits;

		if(type == SF_CONSTANT) {
			bitpos += (uint32_t)sbps;
		}
		else if(type == SF_VERBATIM) {
			// bs raw samples of sbps bits: fixed-width, no scan needed
			const int R = (bs + nthr - 1) / nthr;
			const int i0 = tid * R, i1 = min(bs, i0 + R);
			if(i0 < i1) {
				BitPut bw;
				bw.init(words, bitpos + (uint32_t)i0 * (uint32_t)sbps);
				for(int i = i0; i < i1; i++) bw.put(mask_bits(g[i], (uint32_t)sbps), (uint32_t)sbps);
				bw.finish();
			}
			bitpos += (uint32_t)bs * (uint32_t)sbps;
		}
		else {
			bitpos += (uint32_t)order * (uint32_t)sbps;
			if(type == SF_LPC) bitpos += kQlpPrecisionLen + kQlpShiftLen + (uint32_t)order * (uint32_t)pl->precision;
			bitpos += kEntropyTypeLen + kRiceOrderLen;

			// stage the signal, compute the residual (same arithmetic as k_search)
			for(int i = tid; i < bs; i += nthr) x[skew(i)] = g[i];
			__syncthreads();
			if(type == SF_FIXED) {
				for(int i = order + tid; i < bs; i += nthr) {
					int32_t r;
					switch(order) {
						case 0: r = x[skew(i)]; break;
						case 1: r = x[skew(i)] - x[skew(i - 1)]; break;
						case 2: r = x[skew(i)] - 2 * x[skew(i - 1)] + x[skew(i - 2)]; break;
						case 3: r = x[skew(i)] - 3 * x[skew(i - 1)] + 3 * x[skew(i - 2)] - x[skew(i - 3)]; break;
						default: r = x[skew(i)] - 4 * x[skew(i - 1)] + 6 * x[skew(i - 2)] - 4 * x[skew(i - 3)] + x[skew(i - 4)]; break;
					}
					res[skew(i)] = r;
				}
			}
			else {
				const int shift = pl->shift;
				if(!pl->wide) {
					for(int i = order + tid; i < bs; i += nthr) {
						int32_t sum = 0;
						for(int j = 0; j < order; j++) sum += __ldg(&pl->qlp[j]) * x[skew(i - 1 - j)];
						res[skew(i)] = x[skew(i)] - (sum >> shift);
					}
				}
				else {
					for(int i = order + tid; i < bs; i += nthr) {
						int64_t sum = 0;
						for(int j = 0; j < order; j++) sum += (int64_t)__ldg(&pl->qlp[j]) * (int64_t)x[skew(i - 1 - j)];
						res[skew(i)] = (int32_t)((int64_t)x[skew(i)] - (sum >> shift));
					}
				}
			}
			__syncthreads();

			// partitioned Rice coding (stream_encoder_framing.c:538-594, bitwriter.c:575-706)
			const int po = pl->porder;
			const int psize = bs >> po;
			const uint32_t plen = pl->method ? kRice2ParamLen : kRiceParamLen;
			const int R = (bs - order + nthr - 1) / nthr;
			const int i0 = order + tid * R, i1 = min(bs, i0 + R);
			uint32_t mybits = 0;
			if(i0 < i1) {
				int p = i0 / psize;
				int next = (p + 1) * psize;
				uint32_t k = __ldg(&pl->params[p]);
				for(int i = i0; i < i1; i++) {
					if(i == next) { p++; next += psize; k = __ldg(&pl->params[p]); }
					if(i == p * psize || i == order) mybits += plen;
					const int32_t r = res[skew(i)];
					const uint32_t u = ((uint32_t)r << 1) ^ (uint32_t)(r >> 31);
					mybits += (u >> k) + 1 + k;
				}
			}
			uint32_t total;
			const uint32_t start = block_exclusive_scan_256(mybits, s_warp, &total);
			if(i0 < i1) {
				BitPut bw;
				bw.init(words, bitpos + start);
				int p = i0 / psize;
				int next = (p + 1) * psize;
				uint32_t k = __ldg(&pl->params[p]);
				for(int i = i0; i < i1; i++) {
					if(i == next) { p++; next += psize; k = __ldg(&pl->params[p]); }
					if(i == p * psize || i == order) bw.put(k, plen);
					const int32_t r = res[skew(i)];
					const uint32_t u = ((uint32_t)r << 1) ^ (uint32_t)(r >> 31);
					bw.skip(u >> k);
					bw.put((1u << k) | (u & ((1u << k) - 1u)), k + 1);
				}
				bw.finish();
			}
			bitpos += total;
		}
		__syncthreads();
	}

	// ---- zero-pad to a byte boundary, CRC-16 (stream_encoder.c:3465-3480)
	const uint32_t nbytes = (bitpos + 7) >> 3;
	{
		const uint32_t L = (nbytes + nthr - 1) / nthr;  // bytes per thread, chunks aligned to the END of the frame
		const int64_t cstart = (int64_t)nbytes - (int64_t)(nthr - tid) * L;
		const int64_t cend = cstart + L;
		uint32_t crc = 0;
		for(int64_t b = (cstart < 0 ? 0 : cstart); b < cend; b++) {
			const uint32_t byte = (words[b >> 2] >> (24 - 8 * ((uint32_t)b & 3))) & 0xffu;
			crc = ((crc << 8) & 0xffffu) ^ s_crctab[((crc >> 8) ^ byte) & 0xffu];
		}
		s_crc[tid] = crc;
		if(tid == 0) {
			// x^(8L) mod P by square-and-multiply, then repeated squaring for the tree levels
			uint32_t result = 1, base = 2, e = 8 * L;
			while(e) {
				if(e & 1) result = gf16_mul(result, base);
				base = gf16_mul(base, base);
				e >>= 1;
			}
			for(int s = 0; s < 8; s++) { s_mlev[s] = result; result = gf16_mul(result, result); }
		}
		__syncthreads();
		for(int s = 0; s < 8; s++) {
			if((tid & ((2 << s) - 1)) == 0) s_crc[tid] = gf16_mul(s_crc[tid], s_mlev[s]) ^ s_crc[tid + (1 << s)];
			__syncthreads();
		}
	}
	if(tid == 0) {
		const uint32_t crc = s_crc[0];
		BitPut bw;
		bw.init(words, nbytes * 8);
		bw.put(crc, 16);
		bw.finish();
		frame_bytes[blk] = nbytes + 2;
		if(chan_assign_out) chan_assign_out[blk] = (uint32_t)ca;
	}
	__syncthreads();
	{
		const uint32_t nwords = (nbytes + 2 + 3) >> 2;
		uint32_t *dst = reinterpret_cast<uint32_t *>(slots + (size_t)blk * P.slot_stride);
		for(uint32_t i = tid; i < nwords; i += nthr) dst[i] = __byte_perm(words[i], 0, 0x0123);
	}
}

// ================================================================ k_scan / k_gather
// offsets[first + i] = *running + sum_{j<i} bytes[j]; offsets[first+n] and *running updated.
__global__ void __launch_bounds__(1024) k_scan(const uint32_t *__restrict__ bytes, int n, unsigned long long *__restrict__ offsets,
                                              unsigned long long *__restrict__ running)
{
	__shared__ unsigned long long s_part[1024];
	const int tid = threadIdx.x;
	const int per = (n + 1023) / 1024;
	const int b = tid * per, e = min(n, b + per);
	unsigned long long s = 0;
	for(int i = b; i < e; i++) s += bytes[i];
	s_part[tid] = s;
	__syncthreads();
	// inclusive scan of 1024 partials (Hillis-Steele)
	for(int o = 1; o < 1024; o <<= 1) {
		unsigned long long t = (tid >= o) ? s_part[tid - o] : 0;
		__syncthreads();
		s_part[tid] += t;
		__syncthreads();
	}
	const unsigned long long base = *running;
	unsigned long long acc = base + s_part[tid] - s;
	for(int i = b; i < e; i++) { offsets[i] = acc; acc += bytes[i]; }
	__syncthreads();
	if(tid == 1023) {
		offsets[n] = base + s_part[1023];
		*running = base + s_part[1023];
	}
}

__global__ void __launch_bounds__(256) k_gather(EncK P, const uint8_t *__restrict__ slots, const uint32_t *__restrict__ bytes,
                                               const unsigned long long *__restrict__ offsets, uint8_t *__restrict__ out,
                                               unsigned long long capacity, int *__restrict__ err)
{
	const int blk = blockIdx.x, tid = threadIdx.x;
	const uint32_t n = bytes[blk];
	const unsigned long long off = offsets[blk];
	if(off + n > capacity) {
		if(tid == 0) atomicExch(err, 1);
		return;
	}
	const uint8_t *src = slots + (size_t)blk * P.slot_stride;
	uint8_t *dst = out + off;
	// head bytes up to 4-byte alignment of dst, then word copies assembled from the (aligned) slot
	const uint32_t head = min(n, (uint32_t)((4u - ((uint32_t)(uintptr_t)dst & 3u)) & 3u));  // align on the ADDRESS: `out` itself may be unaligned
	if(tid < head) dst[tid] = src[tid];
	const uint32_t nw = (n - head) >> 2;
	const uint32_t *s32 = reinterpret_cast<const uint32_t *>(src);
	uint32_t *d32 = reinterpret_cast<uint32_t *>(dst + head);
	const uint32_t sh = head * 8;  // source is misaligned by `head` bytes relative to dst words
	for(uint32_t i = tid; i < nw; i += 256) {
		uint32_t v;
		if(sh == 0) v = s32[i];
		else v = __funnelshift_r(s32[i], s32[i + 1], sh);
		d32[i] = v;
	}
	const uint32_t tail0 = head + nw * 4;
	if(tail0 + tid < n) dst[tail0 + tid] = src[tail0 + tid];
}

}  // namespace fb200
