// autoc_kernel.cuh -- k_autoc3: windowed FP64 autocorrelation, one warp per 32 chains,
// samples staged through shared memory with an asynchronous multi-stage copy pipeline.
//
// What bounds this kernel (tools/ubench/fp64_rates.cu measures these rates): the DFMA issue rate,
// the latency of a dependent DFMA, and F2F.F64.F32 on its own, slower pipe.  A chain (one section of
// one signal) must add its lag products in ascending sample order (lpc.c:121-140 sums that way
// and every partial sum is rounded), so the only parallelism is ACROSS chains and across the
// LAGS accumulators of one chain.  One thread therefore owns one chain with all its lags in
// registers (LAGS independent DFMA chains >= the 6 needed to cover the DFMA latency), and the
// job of the rest of the kernel is to keep that thread from ever waiting on memory: k_autoc2
// (thread-private 128-bit global loads, one predicated window load per sample) spent most of
// its cycles waiting on loads, because with at most a few warps per sub-partition nothing
// hides a load.
//
// Layout: CTA = one warp = 32 consecutive items of ONE section (so window indices, tile
// counts and all control flow are warp-uniform).  Per tile of T samples the warp issues
//   * 32 x T/4 16-byte cp.async.cg (each lane: consecutive 16-byte pieces of a row -> 128-byte
//     coalesced segments) into rows of STRIDE words, STRIDE/4 odd => the 128-bit row reads of
//     the 32 lanes (one row each) are bank-conflict free,
//   * T 4-byte cp.async (zero-filled outside the section: the partial windows of
//     lpc.c:82-94 become plain weights) for the window tile, read back as broadcast float4,
// STAGES tiles deep.  The compute loop is branch-free: I2F, FMUL, F2F, LAGS x DFMA per sample.
// fma(d, h, acc) equals the reference's acc += d*h exactly: d and h are floats widened to
// double, so their product is exact in double and only the addition rounds.
#pragma once

#include "device_common.cuh"

namespace fb200 {

__device__ __forceinline__ void cp_async_16(void *smem, const void *gmem)
{
	const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}
// 4-byte copy; src_bytes == 0 writes zeros without touching gmem
__device__ __forceinline__ void cp_async_4_zfill(void *smem, const void *gmem, int src_bytes)
{
	const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// smallest row stride (words) >= T with stride % 4 == 0 and (stride / 4) odd
__host__ __device__ constexpr int autoc3_stride(int T) { return ((T / 4) % 2 == 1) ? T : T + 4; }
template <int LAGS, int U, int K, int STAGES>
constexpr size_t autoc3_smem_bytes() { return (size_t)STAGES * (32 * autoc3_stride(U * K) + U * K) * 4; }

template <int LAGS, int U, int K, int STAGES>
__global__ void __launch_bounds__(32) k_autoc3(EncK P, const int32_t *__restrict__ sig, const SigMeta *__restrict__ meta,
                                              const float *__restrict__ windows, const DevSection *__restrict__ secs,
                                              double *__restrict__ autoc, int nitems)
{
	static_assert(U % LAGS == 0 && U % 4 == 0, "a body must be a whole number of history rotations and of 128-bit loads");
	constexpr int T = U * K;
	constexpr int STRIDE = autoc3_stride(T);
	constexpr int STAGE_WORDS = 32 * STRIDE + T;
	extern __shared__ int4 autoc3_smem[];
	int *const smem = reinterpret_cast<int *>(autoc3_smem);

	const int lane = threadIdx.x;
	// section slowest: the longest chains (full-length sections) start first. (Section-fastest ordering would let L2
	// serve the partial-window re-reads, which multiply DRAM traffic at -8, but it was measured slower on the GPU this
	// kernel was first tuned on, not on H100: the kernel is FP64-bound and the long chains then finish last.)
	const int groups = (nitems + 31) >> 5;
	const int sec = blockIdx.x / groups;
	const int item0 = (blockIdx.x - sec * groups) << 5;
	const int item = item0 + lane;
	const bool live = item < nitems && meta[min(item, nitems - 1)].bps != 0;
	if(!__any_sync(0xffffffffu, live)) return;

	const DevSection S = secs[sec];
	const float *w = windows + S.win_off;
	const int shift = S.partial ? S.data_shift : 0;
	const int a0 = shift & ~3;                                    // 16-byte aligned first sample fetched
	const int nvalid = S.partial ? 2 * S.part_size : S.data_len;  // weights are 0 from here on (lpc.c:90-91): nothing to add
	const int wsecond = P.bs - 2 * S.part_size;                   // window index offset of the falling half
	const int ntiles = (shift - a0 + nvalid + T - 1) / T;

	auto issue = [&](int t) {
		if(t < ntiles) {
			int *st = smem + (t % STAGES) * STAGE_WORDS;
			const int32_t *g0 = sig + a0 + t * T;
#pragma unroll
			for(int j = 0; j < T / 4; j++) {
				const int idx = j * 32 + lane;
				const int row = idx / (T / 4), c = idx - row * (T / 4);
				cp_async_16(st + row * STRIDE + c * 4, g0 + (size_t)min(item0 + row, nitems - 1) * P.bs_stride + c * 4);
			}
#pragma unroll
			for(int j = 0; j < (T + 31) / 32; j++) {
				const int u = j * 32 + lane;
				if(u < T) {
					const int i = a0 + t * T + u - shift;  // index inside the section
					const bool ok = i >= 0 && i < nvalid;
					const int wi = (!S.partial || i < S.part_size) ? i : wsecond + i;
					cp_async_4_zfill(st + 32 * STRIDE + u, ok ? (w + wi) : w, ok ? 4 : 0);
				}
			}
		}
		cp_async_commit();  // one group per call, empty or not, keeps wait_group's count aligned with t
	};

	double acc[LAGS], h[LAGS];
#pragma unroll
	for(int l = 0; l < LAGS; l++) { acc[l] = 0.0; h[l] = 0.0; }

#pragma unroll
	for(int t = 0; t < STAGES - 1; t++) issue(t);
	for(int t = 0; t < ntiles; t++) {
		cp_async_wait<STAGES - 2>();  // tile t has landed (this lane's copies) ...
		__syncwarp();                 // ... and every other lane's; all lanes are also done with tile t-1's buffer
		issue(t + STAGES - 1);
		const int *row = smem + (t % STAGES) * STAGE_WORDS + lane * STRIDE;
		const float *win = reinterpret_cast<const float *>(smem + (t % STAGES) * STAGE_WORDS + 32 * STRIDE);
#pragma unroll 1
		for(int kb = 0; kb < K; kb++) {
#pragma unroll
			for(int q = 0; q < U / 4; q++) {
				const int4 xq = *reinterpret_cast<const int4 *>(row + kb * U + q * 4);
				const float4 wq = *reinterpret_cast<const float4 *>(win + kb * U + q * 4);
				const int xs[4] = {xq.x, xq.y, xq.z, xq.w};
				const float ws[4] = {wq.x, wq.y, wq.z, wq.w};
#pragma unroll
				for(int e = 0; e < 4; e++) {
					const int u = q * 4 + e;
					const double dv = (double)__fmul_rn((float)xs[e], ws[e]);  // lpc.c:68-74: float product, widened
					const int su = (LAGS - (u % LAGS)) % LAGS;                  // slot of the newest sample; slot (su+l)%LAGS holds d[i-l]
					h[su] = dv;
#pragma unroll
					for(int l = 0; l < LAGS; l++) acc[l] = fma(dv, h[(su + l) % LAGS], acc[l]);
				}
			}
		}
	}
	if(live) {
		double *out = autoc + ((size_t)sec * nitems + item) * P.lag_stride;
#pragma unroll
		for(int l = 0; l < LAGS; l++) out[l] = acc[l];
	}
}


// ================================================================ k_autoc4
// The same chain-per-thread scheme fed from the CALLER'S interleaved int32 PCM (no planar copy): the warp's 32 chains
// are 32 consecutive (block, signal) items of one section, i.e. a handful of blocks; per tile the raw rows of those
// blocks (T samples x channels) and the section's weight tile are staged with 1-D TMA bulk copies onto an mbarrier
// ring (cp.async.bulk + mbarrier::complete_tx: one copy per block row instead of T/4 16-byte cp.async per lane), and
// every lane derives ITS signal from the raw row on the fly: channel c, or mid = (L+R)>>1 / side = L-R
// (stream_encoder.c:3823-3836), wasted bits shifted out (:3842-3867). The per-section weight table (host-built,
// zero outside the section) turns the partial windows of lpc.c:82-94 into plain weights.
// MODE 0: mono (128-bit row reads = 4 samples); 1: two channels (128-bit = 2 sample pairs, signal = (a L + b R) >> sh);
// 2: any channel count (scalar reads).
__host__ __device__ constexpr int autoc4_rows_max(int nsig) { return (nsig + 30) / nsig + 1; }
__host__ __device__ constexpr int autoc4_row_stride(int T, int ch, int mode)
{
	// words; multiples of 4 (TMA destination alignment); modes 0/1: an odd number of 16-byte units -> the 128-bit reads
	// of distinct rows fall into distinct bank groups; mode 2: rows 8 banks apart
	return mode == 2 ? T * ch + 8 : (((T * ch / 4) & 1) ? T * ch : T * ch + 4);
}
template <int U, int K, int STAGES>
__host__ __device__ constexpr size_t autoc4_smem_bytes(int nsig, int ch, int mode)
{
	return 64 + (size_t)STAGES * ((size_t)autoc4_rows_max(nsig) * autoc4_row_stride(U * K, ch, mode) + U * K) * 4;
}

template <int LAGS, int U, int K, int STAGES, int MODE>
__global__ void __launch_bounds__(32) k_autoc4(EncK P, const int32_t *__restrict__ pcm, const SigMeta *__restrict__ meta,
                                              const float *__restrict__ secwin, int secwin_stride, const DevSection *__restrict__ secs,
                                              double *__restrict__ autoc, int nitems, uint32_t *__restrict__ sigor, int or_sec)
{
	static_assert(U % LAGS == 0 && U % 4 == 0, "a body must be a whole number of history rotations and of 128-bit loads");
	constexpr int T = U * K;
	extern __shared__ int4 autoc4_smem[];
	uint64_t *const bars = reinterpret_cast<uint64_t *>(autoc4_smem);  // STAGES mbarriers in the first 64 bytes
	int *const smem = reinterpret_cast<int *>(autoc4_smem) + 16;
	const int lane = threadIdx.x, nsig = P.nsig, ch = P.channels, bs = P.bs;
	const int RS = autoc4_row_stride(T, ch, MODE);
	const int STAGE_WORDS = autoc4_rows_max(nsig) * RS + T;

	// section slowest: the longest chains (full-length sections) start first (see k_autoc3)
	const int groups = (nitems + 31) >> 5;
	const int sec = blockIdx.x / groups;
	// sigor: the chains of section or_sec (a full-length one) also OR their samples together -- all get_wasted_bits_ needs
	// (stream_encoder.c:5077-5099); k_lpc turns the word into the signal's wasted bits / subframe bps, and no kernel has to
	// read the block just for that
	const bool do_or = sigor != nullptr && sec == or_sec;
	uint32_t orv = 0;
	const int item0 = (blockIdx.x - sec * groups) << 5;
	const int item = min(item0 + lane, nitems - 1);
	// meta == nullptr: the wasted-bits shift is left to k_lpc (the windowed products and their sums scale EXACTLY by powers of
	// two, so autoc(x >> w) == autoc(x) * 2^-2w bit for bit) and every signal is analysed -- k_meta then runs concurrently
	SigMeta M;
	M.wasted = 0; M.bps = 1;
	if(meta) M = meta[item];
	const bool live = item0 + lane < nitems && M.bps != 0;
	if(!__any_sync(0xffffffffu, live)) return;

	const DevSection S = secs[sec];
	const int shift = S.partial ? S.data_shift : 0;
	const int a0 = shift & ~3;                                    // 16-byte aligned first sample fetched
	const int nvalid = S.partial ? 2 * S.part_size : S.data_len;  // weights are 0 from here on (lpc.c:90-91): nothing to add
	const int ntiles = (shift - a0 + nvalid + T - 1) / T;
	const int b0 = item0 / nsig;
	const int nrows = min(item0 + 31, nitems - 1) / nsig - b0 + 1;
	const int myrow = item / nsig - b0, sidx = item - (item / nsig) * nsig;
	const float *wsec = secwin + (size_t)sec * secwin_stride;

	// this lane's signal as (a * X + b * Y) >> sh of the raw row; X = channel c0, Y = channel 1 (two-channel mode only)
	int ca = 1, cb = 0, sh = M.wasted;
	if(MODE == 1) {
		if(sidx == 1) { ca = 0; cb = 1; }
		else if(sidx == 2) { ca = 1; cb = 1; sh += 1; }
		else if(sidx == 3) { ca = 1; cb = -1; }
	}

	if(lane == 0) {
#pragma unroll
		for(int s = 0; s < STAGES; s++) mbar_init(&bars[s], 1);
		mbar_fence_init();
	}
	__syncwarp();

	auto issue = [&](int t) {
		if(t < ntiles) {
			const int stg = t % STAGES;
			int *st = smem + stg * STAGE_WORDS;
			const int start = a0 + t * T;
			const int n = min(T, bs - start);  // never read past the block (the last block ends the caller's buffer)
			const unsigned row_bytes = (unsigned)n * (unsigned)ch * 4u;
			if(lane == 0) mbar_expect_tx(&bars[stg], (unsigned)nrows * row_bytes + (unsigned)T * 4u);
			__syncwarp();
			if(lane < nrows) tma_bulk_g2s(st + lane * RS, pcm + ((size_t)(b0 + lane) * bs + start) * ch, row_bytes, &bars[stg]);
			if(lane == (nrows < 32 ? nrows : 0)) tma_bulk_g2s(st + autoc4_rows_max(nsig) * RS, wsec + start, (unsigned)T * 4u, &bars[stg]);  // the table has T zeros of slack
		}
	};

	double acc[LAGS], h[LAGS];
#pragma unroll
	for(int l = 0; l < LAGS; l++) { acc[l] = 0.0; h[l] = 0.0; }

#pragma unroll
	for(int t = 0; t < STAGES - 1; t++) issue(t);
	for(int t = 0; t < ntiles; t++) {
		__syncwarp();                 // every lane is done with tile t-1's buffer ...
		issue(t + STAGES - 1);        // ... which is the one refilled now
		mbar_wait(&bars[t % STAGES], (unsigned)(t / STAGES) & 1u);
		if(do_or && bs - (a0 + t * T) < T) {
			// the block's last tile is short: what lies behind it in the buffer is stale, weighted 0 in the sums but not in the OR
			const int n = bs - (a0 + t * T);
			int *st = smem + (t % STAGES) * STAGE_WORDS;
			for(int r = 0; r < nrows; r++)
				for(int i = n * ch + lane; i < T * ch; i += 32) st[r * RS + i] = 0;
			__syncwarp();
		}
		const int *row = smem + (t % STAGES) * STAGE_WORDS + myrow * RS;
		const float *win = reinterpret_cast<const float *>(smem + (t % STAGES) * STAGE_WORDS + autoc4_rows_max(nsig) * RS);
#pragma unroll 1
		for(int kb = 0; kb < K; kb++) {
#pragma unroll
			for(int q = 0; q < U / 4; q++) {
				int xs4[4];
				if(MODE == 0) {
					const int4 xq = *reinterpret_cast<const int4 *>(row + kb * U + q * 4);
					xs4[0] = xq.x >> sh; xs4[1] = xq.y >> sh; xs4[2] = xq.z >> sh; xs4[3] = xq.w >> sh;
				}
				else if(MODE == 1) {
					const int4 p0 = *reinterpret_cast<const int4 *>(row + 2 * (kb * U + q * 4));
					const int4 p1 = *reinterpret_cast<const int4 *>(row + 2 * (kb * U + q * 4) + 4);
					xs4[0] = (ca * p0.x + cb * p0.y) >> sh; xs4[1] = (ca * p0.z + cb * p0.w) >> sh;
					xs4[2] = (ca * p1.x + cb * p1.y) >> sh; xs4[3] = (ca * p1.z + cb * p1.w) >> sh;
				}
				else {
#pragma unroll
					for(int e = 0; e < 4; e++) xs4[e] = row[(kb * U + q * 4 + e) * ch + sidx] >> sh;
				}
				const float4 wq = *reinterpret_cast<const float4 *>(win + kb * U + q * 4);
				const float ws[4] = {wq.x, wq.y, wq.z, wq.w};
				orv |= (uint32_t)(xs4[0] | xs4[1]) | (uint32_t)(xs4[2] | xs4[3]);
#pragma unroll
				for(int e = 0; e < 4; e++) {
					const int u = q * 4 + e;
					const double dv = (double)__fmul_rn((float)xs4[e], ws[e]);  // lpc.c:68-74: float product, widened
					const int su = (LAGS - (u % LAGS)) % LAGS;                   // slot of the newest sample; slot (su+l)%LAGS holds d[i-l]
					h[su] = dv;
#pragma unroll
					for(int l = 0; l < LAGS; l++) acc[l] = fma(dv, h[(su + l) % LAGS], acc[l]);
				}
			}
		}
	}
	if(live) {
		double *out = autoc + ((size_t)sec * nitems + item) * P.lag_stride;
#pragma unroll
		for(int l = 0; l < LAGS; l++) out[l] = acc[l];
		if(do_or) sigor[item] = orv;
	}
}

}  // namespace fb200
