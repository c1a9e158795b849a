// search_kernel.cuh -- k_search5: one CTA per block, two warps per signal, register-resident partition tree.
//
// Profiling k_search3 at -8 showed the FIR taps taking the smaller part of the time; most went into
// the per-candidate tail (zeroing / read-modify-write of a shared-memory heap, six barrier-separated
// merge levels, four chunked parameter sweeps with 64-bit shared traffic) and into group-loop control
// (a jump-table switch and dozens of address instructions per 16-output group).  This generation keeps the arithmetic and the
// decision order (stream_encoder.c:4191-4269, 4701-5075) and changes the mechanics:
//   * the predictor class (taps x width) is chosen ONCE per candidate; the tile/group loops are
//     straight pointer walks (a zeroed row in front of the signal removes the row-0 branch);
//   * a run's |residual| sum goes to its leaf with a plain store (no zeroing, no RMW, no barrier);
//   * the partition tree lives in registers: a lane owns 2^(max_po-5) consecutive leaves, merges
//     them locally down to order 5 and continues with xor-shuffles; Rice parameter and bit count
//     of a node are computed where the node lives; an order's total is one warp reduction;
//     the best order is tracked in registers while walking the orders downwards.
#pragma once

#include "device_common.cuh"

namespace fb200 {

// The 64-bit-accumulator predictor (lpc.c:786-884, subframes deeper than 16 bits) on the FP64 pipe: IMAD.WIDE
// chains issue several times slower than DFMA (tools/ubench measures both). Everything here is an integer
// below 2^51 held in a double, so every operation is exact: qd[j] = q[j] * 2^-shift (a power-of-two scaling keeps
// the significand), sum = sum_j qd[j] x[i-1-j] = (integer sum) / 2^shift, floor(sum) by adding 1.5 * 2^52 rounding
// down (== the reference's arithmetic right shift), |residual| added into a double (< 2^45 per run).
template <int G, int MAXORD, int NTAPS, bool MASKED>
__device__ __forceinline__ void group_abs_sum_f64(const int (&xg)[MAXORD + G], const double (&qd)[MAXORD], int ord0, int limit, double &sd, bool &bad)
{
	constexpr double kFloorMagic = 6755399441055744.0;  // 1.5 * 2^52
	double xd[MAXORD + G];
#pragma unroll
	for(int i = MAXORD - NTAPS; i < MAXORD + G; i++) xd[i] = int_to_double_exact(xg[i]);
#pragma unroll
	for(int m = 0; m < G; m++) {
		double sum = 0.0;
#pragma unroll
		for(int j = 0; j < NTAPS; j++) sum = fma(qd[j], xd[MAXORD + m - 1 - j], sum);
		const double t = __dadd_rd(sum, kFloorMagic);                          // floor(sum) + magic
		const double rr = __dadd_rn(__dsub_rn(xd[MAXORD + m], t), kFloorMagic);  // x - floor(sum): the residual
		if(limit && (rr <= -2147483648.0 || rr > 2147483647.0)) bad = true;    // lpc.c:868-884
		bool keep = true;
		if(MASKED && m < MAXORD) keep = m >= ord0;
		if(keep) sd = __dadd_rn(sd, fabs(rr));
	}
}

// All runs of one candidate: leaf[p] = sum of |residual| over finest partition p.
// xs = first sample of the warp's slice (row stride 36 words, kSearch4ZeroRow zero words in front).
// lpp_log: log2(lanes per partition) when a partition fits in a tile (tpp == 1), else tpp tiles make one partition.
// Returns true when a wide residual left the int32 range (lpc.c:868-884).
template <int R_T, int MAXORD, int NTAPS, bool WIDE, bool NARROW>
__device__ __forceinline__ bool fir_partition_sums(const int32_t *xs, const int (&q)[MAXORD], int shift, int order, int limit,
                                                   int ntiles, int lane, int lpp_log, int tpp, bool mask32, unsigned long long *leaf)
{
	constexpr int G = (R_T == 32) ? 16 : 12, NG = R_T / G, ROWPAD = 36 - R_T;
	bool bad = false;
	unsigned long long carry = 0;
	double qd[MAXORD];
	if(WIDE) {
		const double scale = __hiloint2double((1023 - shift) << 20, 0);  // 2^-shift
#pragma unroll
		for(int j = 0; j < MAXORD; j++) qd[j] = __dmul_rn((double)q[j], scale);
	}
	// The pass below treats every sample as a residual (one code path, half the instruction footprint of a
	// masked first tile). The first `order` outputs of the block are warm-up samples, not residuals: their
	// |"residual"| (history before the block = the zero row) is recomputed here and taken out of partition 0.
	unsigned long long warm = 0;
	{
		int xw[MAXORD];
#pragma unroll
		for(int k = 0; k < MAXORD / 4; k++) {
			const int4 v = *reinterpret_cast<const int4 *>(xs + 4 * k);
			xw[4 * k] = v.x; xw[4 * k + 1] = v.y; xw[4 * k + 2] = v.z; xw[4 * k + 3] = v.w;
		}
#pragma unroll
		for(int m = 0; m < MAXORD; m++) {
			unsigned long long a;
			if(!WIDE) {
				int sum = 0;
#pragma unroll
				for(int j = 0; j < (m < NTAPS ? m : NTAPS); j++) sum += q[j] * xw[m - 1 - j];
				a = __sad(xw[m], sum >> shift, 0u);
			}
			else {
				long long sum = 0;
#pragma unroll
				for(int j = 0; j < (m < NTAPS ? m : NTAPS); j++) sum += (long long)q[j] * (long long)xw[m - 1 - j];
				const long long rr = (long long)xw[m] - (sum >> shift);
				a = (unsigned long long)(rr < 0 ? -rr : rr);
			}
			if(m < order) warm += a;
		}
	}
#pragma unroll 1
	for(int t = 0; t < ntiles; t++) {
		const int32_t *rowp = xs + (t * 32 + lane) * 36;
		uint32_t s32 = 0;
		unsigned long long s64 = 0;
		double sd = 0.0;
#pragma unroll 1
		for(int g = 0; g < NG; g++) {
			int xg[MAXORD + G];
			const int32_t *op = rowp + g * G;                               // first output of the group
			// history vector k holds samples [g*G - MAXORD + 4k, +4) of the run; negative ones live in the previous row,
			// i.e. behind the row pad (MAXORD <= R_T, so never further than one row back)
#pragma unroll
			for(int k = 0; k < MAXORD / 4; k++) {
				const int4 v = *reinterpret_cast<const int4 *>(op - MAXORD + 4 * k - ((g * G + 4 * k < MAXORD) ? ROWPAD : 0));
				xg[4 * k] = v.x; xg[4 * k + 1] = v.y; xg[4 * k + 2] = v.z; xg[4 * k + 3] = v.w;
			}
#pragma unroll
			for(int k = 0; k < G / 4; k++) {
				const int4 v = *reinterpret_cast<const int4 *>(op + 4 * k);
				xg[MAXORD + 4 * k] = v.x; xg[MAXORD + 4 * k + 1] = v.y; xg[MAXORD + 4 * k + 2] = v.z; xg[MAXORD + 4 * k + 3] = v.w;
			}
			if(WIDE) group_abs_sum_f64<G, MAXORD, NTAPS, false>(xg, qd, 0, limit, sd, bad);
			else group_abs_sum<G, MAXORD, NTAPS, false, false, NARROW>(xg, q, shift, 0, limit, s32, s64, bad);
		}
		if(WIDE) s64 = (unsigned long long)__double2ll_rn(sd);  // an exact non-negative integer
		if(tpp == 1) {
			const int lpp = 1 << lpp_log;
			if(NARROW) {
				uint32_t s = s32;  // the reference's 32-bit accumulator wraps (stream_encoder.c:4815-4824); so does this
				for(int o = lpp >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
				if(t == 0 && lane == 0) s -= (uint32_t)warm;
				if((lane & (lpp - 1)) == 0) leaf[(t * 32 + lane) >> lpp_log] = s;
			}
			else {
				unsigned long long s = s64;
				for(int o = lpp >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
				if(t == 0 && lane == 0) s -= warm;
				if((lane & (lpp - 1)) == 0) leaf[(t * 32 + lane) >> lpp_log] = mask32 ? (unsigned long long)(uint32_t)s : s;
			}
		}
		else {
			carry += warp_sum_u64(NARROW ? (unsigned long long)s32 : s64);
			if(t + 1 == tpp) carry -= warm;
			if((t + 1) % tpp == 0) {
				if(lane == 0) leaf[t / tpp] = (NARROW || mask32) ? (unsigned long long)(uint32_t)carry : carry;
				carry = 0;
			}
		}
	}
	return bad;
}

// What one warp found for its signal (second warp of a signal -> first warp, through shared memory).
struct SearchResult5 {
	uint32_t best_bits;
	int idx, type, order, prec, shift, method, po, wide, pad;
	int q[FB200_MAX_LPC_ORDER];
};

__host__ __device__ constexpr size_t search5_scratch_bytes(int max_po)
{
	// per warp: leaf[2^max_po] u64, params_all[2 * 2^max_po] u8, b_params[2^max_po] u8 -- rounded to 16 bytes
	return (((size_t)8 << max_po) + ((size_t)3 << max_po) + 15) / 16 * 16;
}
__host__ __device__ constexpr size_t search5_smem_bytes(int bs, int R_T, int nsig, int wps, int max_po)
{
	return (size_t)nsig * (size_t)(kSearch4ZeroRow + (bs / R_T) * 36) * 4 + (size_t)nsig * wps * search5_scratch_bytes(max_po) +
	       (size_t)nsig * (sizeof(SearchResult5) + 16) + 64 + (size_t)nsig * 48;
}

// One CTA per block. Shared memory: nsig signal slices (row layout: 36-word rows, a zero row in front), filled ONCE per
// block from the caller's interleaved int32 PCM -- 1-2 channels: one TMA bulk copy of the raw block, pulled into registers
// and written back as L / R / mid / side slices in place; more channels: strided gather -- then WPS warps per signal share
// the signal's slice and split its candidates: warp 0 runs the fixed-predictor scan and the fixed candidate(s), every warp
// takes LPC candidates from a per-signal queue (atomic counter). Each warp keeps its own first-minimum (strict '<' in
// evaluation order, stream_encoder.c:4191-4269); the merge takes the smaller estimate and, on a tie, the smaller
// candidate index -- i.e. exactly the candidate the reference's sequential best-of-two keeps.
template <int R_T, int MAXORD, int WPS, bool WIDEK>
__global__ void __launch_bounds__(256, 2) k_search5(EncK P, const int32_t *__restrict__ pcm, const SigMeta *__restrict__ meta,
                                                    const CandDesc *__restrict__ cdesc, SubframePlan *__restrict__ plans)
{
	static_assert(MAXORD >= 8 && MAXORD % 4 == 0 && R_T % 4 == 0 && MAXORD + 4 <= kSearch4ZeroRow, "vector loads / zero row");
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int tid = threadIdx.x, NT = blockDim.x, warp = tid >> 5, lane = tid & 31, bs = P.bs, ch = P.channels;
	// P.sig_group > 0 (more than four signals): a block's signals are split over several CTAs of sig_group signals each -- half
	// the shared memory per CTA, twice the warps per SM; `nsig` below is this CTA's share, sig0 its first signal
	const int ngroups = P.sig_group ? (P.nsig + P.sig_group - 1) / P.sig_group : 1;
	const int blk = (int)blockIdx.x / ngroups;
	const int sig0 = P.sig_group ? ((int)blockIdx.x - blk * ngroups) * P.sig_group : 0;
	const int nsig = P.sig_group ? min(P.sig_group, P.nsig - sig0) : P.nsig;
	if(P.redo && !P.redo[blk]) return;  // second pass of limit_min_bitrate: flagged blocks only
	const int nrows = bs / R_T;
	const int slice_words = kSearch4ZeroRow + nrows * 36;
	int32_t *const slices = reinterpret_cast<int32_t *>(smem_raw);
	unsigned char *const scratch0 = smem_raw + (size_t)nsig * slice_words * 4;
	const size_t scratch_bytes = search5_scratch_bytes(P.max_po);
	unsigned char *const after_scratch = scratch0 + (size_t)nsig * WPS * scratch_bytes;
	SearchResult5 *const results = reinterpret_cast<SearchResult5 *>(after_scratch);
	int *const queues = reinterpret_cast<int *>(after_scratch + (size_t)nsig * sizeof(SearchResult5));
	uint64_t *const mbar = reinterpret_cast<uint64_t *>(queues + nsig + (nsig & 1));  // 8-byte aligned: nsig + pad ints after 16-byte aligned results
	unsigned long long *const xch_all = reinterpret_cast<unsigned long long *>(mbar + 1);  // [nsig][6]: partial scan sums of a signal's second warp

	const SigMeta *bm = meta + (size_t)blk * P.nsig + sig0;
	const bool stereo_ms = (ch == 2 && P.nsig == 4);

	// ---- stage the block: raw interleaved PCM -> planar slices
	if(tid < nsig) queues[tid] = 0;
	const int32_t *graw = pcm + (size_t)blk * bs * ch;
	if(ch <= 2 && (bs * ch) % (4 * NT) == 0 && (bs * ch / 4) / NT <= 16) {
		const unsigned raw_bytes = (unsigned)bs * (unsigned)ch * 4u;
		// the raw block lands behind the zero row of slice 0 ... inside the slice area, which is at least as large
		int32_t *const raw = slices + kSearch4ZeroRow + ((nsig * slice_words - kSearch4ZeroRow - bs * ch) & ~3);
		if(tid == 0) {
			mbar_init(mbar, 1);
			mbar_fence_init();
			mbar_expect_tx(mbar, raw_bytes);
			tma_bulk_g2s(raw, graw, raw_bytes, mbar);
		}
		__syncthreads();
		mbar_wait(mbar, 0);
		int4 rv[16];
		const int nv = (bs * ch / 4) / NT;
#pragma unroll
		for(int k = 0; k < 16; k++)
			if(k < nv) rv[k] = *reinterpret_cast<const int4 *>(raw + 4 * (k * NT + tid));
		__syncthreads();  // the raw block is in registers: the slice area may be overwritten
		for(int s = warp; s < nsig; s += NT >> 5)
			for(int i = lane; i < kSearch4ZeroRow; i += 32) slices[s * slice_words + i] = 0;  // history of row 0
		if(ch == 2) {
			const int w0 = bm[0].wasted, w1 = bm[1].wasted;
			const int w2 = stereo_ms ? bm[2].wasted : 0, w3 = stereo_ms ? bm[3].wasted : 0;
			int32_t *const p0 = slices + kSearch4ZeroRow, *const p1 = p0 + slice_words, *const p2 = p1 + slice_words, *const p3 = p2 + slice_words;
#pragma unroll
			for(int k = 0; k < 16; k++)
				if(k < nv) {
					const int i = 2 * (k * NT + tid);
					const int row = i / R_T, off = row * 36 + (i - row * R_T);
					const int L0 = rv[k].x, R0 = rv[k].y, L1 = rv[k].z, R1 = rv[k].w;
					*reinterpret_cast<int2 *>(p0 + off) = make_int2(L0 >> w0, L1 >> w0);
					*reinterpret_cast<int2 *>(p1 + off) = make_int2(R0 >> w1, R1 >> w1);
					if(stereo_ms) {  // mid/side are formed from the unshifted channels (stream_encoder.c:3823-3867)
						*reinterpret_cast<int2 *>(p2 + off) = make_int2(((L0 + R0) >> 1) >> w2, ((L1 + R1) >> 1) >> w2);
						*reinterpret_cast<int2 *>(p3 + off) = make_int2((L0 - R0) >> w3, (L1 - R1) >> w3);
					}
				}
		}
		else {
			const int w0 = bm[0].wasted;
			int32_t *const p0 = slices + kSearch4ZeroRow;
#pragma unroll
			for(int k = 0; k < 16; k++)
				if(k < nv) {
					const int i = 4 * (k * NT + tid);
					const int row = i / R_T, off = row * 36 + (i - row * R_T);
					*reinterpret_cast<int4 *>(p0 + off) = make_int4(rv[k].x >> w0, rv[k].y >> w0, rv[k].z >> w0, rv[k].w >> w0);
				}
		}
	}
	else {
		// more than two channels (or an odd geometry): every warp gathers whole signals straight from global memory;
		// the strided reads of one block hit the same lines from all of its warps (L1 / L2 serve them)
		for(int s = warp; s < nsig; s += NT >> 5) {
			const int w = bm[s].wasted;
			int32_t *const ps = slices + s * slice_words + kSearch4ZeroRow;
			for(int i = lane; i < kSearch4ZeroRow; i += 32) ps[i - kSearch4ZeroRow] = 0;  // history of row 0
			for(int i = lane; i < bs; i += 32) {
				int v;
				if(stereo_ms && s >= 2) {
					const int L = __ldg(graw + 2 * i), R = __ldg(graw + 2 * i + 1);
					v = s == 2 ? ((L + R) >> 1) : (L - R);
				}
				else v = __ldg(graw + (size_t)i * ch + sig0 + s);
				const int row = i / R_T;
				ps[row * 36 + (i - row * R_T)] = v >> w;
			}
		}
	}
	__syncthreads();

	// ---- this warp's signal and role
	const int sidx = warp / WPS, part = warp - sidx * WPS;
	const bool have_signal = sidx < nsig;
	const bool skip_sig = P.redo != nullptr && sig0 + sidx < ch - 1;  // second pass: these signals keep their plan
	const SigMeta M = have_signal ? bm[sidx] : SigMeta{0, 0};
	const bool active = have_signal && M.bps != 0 && !skip_sig;
	const int32_t *const xs = slices + (have_signal ? sidx : 0) * slice_words + kSearch4ZeroRow;
	unsigned char *const my_scratch = scratch0 + (size_t)(have_signal ? warp : 0) * scratch_bytes;
	unsigned long long *const leaf = reinterpret_cast<unsigned long long *>(my_scratch);
	uint8_t *const params_all = my_scratch + ((size_t)8 << P.max_po);
	uint8_t *const b_params = params_all + ((size_t)2 << P.max_po);
	const int sbps = M.bps, wasted = M.wasted;

	constexpr int TILE = 32 * R_T;
	constexpr int GAPV = (R_T == 32 ? 4 : 0) / 4;  // pad int4s between a row's history and its start
	const int ntiles = bs / TILE;

	// best-so-far of THIS warp (uniform across the warp); b_idx orders candidates: -1 verbatim baseline, 0..4 fixed orders, 5+c LPC slot c
	uint32_t best_bits = 0xffffffffu;
	int b_idx = -1, b_type = SF_VERBATIM, b_order = 0, b_prec = 0, b_shift = 0, b_method = 0, b_po = 0, b_wide = 0;
	int b_q[MAXORD];
#pragma unroll
	for(int j = 0; j < MAXORD; j++) b_q[j] = 0;
	bool is_constant = false;

	if(active) {
		for(int p = lane; p < (1 << P.max_po); p += 32) b_params[p] = 0;
		if(!(P.dis_verb && bs >= (int)kMaxFixedOrder)) best_bits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)bs * (uint32_t)sbps;
		__syncwarp();

		auto evaluate = [&](int cand_index, int type, int order, int precision, int shift, int wide, int limit, const int (&q)[MAXORD]) {
			int max_po = P.max_po;
			while(max_po > 0 && (bs >> max_po) <= order) max_po--;
			const int min_po = min(P.min_po, max_po);
			const int psize = bs >> max_po;
			const bool narrow = (uint32_t)(sbps + (int)kMaxExtraResidualBps) < 32u - ilog2_u32((uint32_t)psize);
			const int tpp = psize > TILE ? psize / TILE : 1;
			const int lpp_log = tpp == 1 ? (int)ilog2_u32((uint32_t)(psize / R_T)) : 5;

			// ---- residual pass, one predictor class per candidate
			constexpr int NT12 = MAXORD < 12 ? MAXORD : 12;
			bool bad = false;
			// The second warp of a signal runs its candidates on the FP64 pipe even when 32-bit accumulation would do (exact: every
			// value is an integer below 2^52): the IMAD pipe is half rate and the first warp keeps it busy, the DFMA pipe is idle
			const bool via_f64 = wide || (WIDEK && WPS == 2 && part == 1 && P.f64b != 0);
			if(!via_f64 && narrow) {
				if(order <= 4) bad = fir_partition_sums<R_T, MAXORD, 4, false, true>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, true, leaf);
				else if(order <= 8) bad = fir_partition_sums<R_T, MAXORD, 8, false, true>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, true, leaf);
				else if(MAXORD > 8 && order <= 12) bad = fir_partition_sums<R_T, MAXORD, NT12, false, true>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, true, leaf);
				else bad = fir_partition_sums<R_T, MAXORD, MAXORD, false, true>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, true, leaf);
			}
			else if(!via_f64) {
				if(order <= 8) bad = fir_partition_sums<R_T, MAXORD, 8, false, false>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, narrow, leaf);
				else if(MAXORD > 8 && order <= 12) bad = fir_partition_sums<R_T, MAXORD, NT12, false, false>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, narrow, leaf);
				else bad = fir_partition_sums<R_T, MAXORD, MAXORD, false, false>(xs, q, shift, order, 0, ntiles, lane, lpp_log, tpp, narrow, leaf);
			}
			else if(WIDEK) {
				if(order <= 8) bad = fir_partition_sums<R_T, MAXORD, 8, true, false>(xs, q, shift, order, limit, ntiles, lane, lpp_log, tpp, narrow, leaf);
				else if(MAXORD > 8 && order <= 12) bad = fir_partition_sums<R_T, MAXORD, NT12, true, false>(xs, q, shift, order, limit, ntiles, lane, lpp_log, tpp, narrow, leaf);
				else bad = fir_partition_sums<R_T, MAXORD, MAXORD, true, false>(xs, q, shift, order, limit, ntiles, lane, lpp_log, tpp, narrow, leaf);
			}
			else bad = fir_partition_sums<R_T, MAXORD, MAXORD, true, false>(xs, q, shift, order, limit, ntiles, lane, lpp_log, tpp, narrow, leaf);
			if(__any_sync(0xffffffffu, bad)) return;  // evaluate_lpc_subframe_ returns 0 (stream_encoder.c:4601-4609)
			__syncwarp();

			// ---- partition orders max_po .. min_po (find_best_partition_order_, :4701-4795; set_partitioned_rice_, :4954-5075)
			uint32_t best_r = 0;
			int best_po = 0;
			const uint32_t rice_cap = (uint32_t)P.rice_limit - 1;
			// Rice parameter (:4994-5010) + bit count (:4929-4951) of heap node n holding `mean`; stores the parameter when `own`
			auto node_bits = [&](unsigned long long mean, uint32_t psamp, uint32_t div, int n, bool own) -> uint32_t {
				uint32_t k;
				if((mean >> 32) == 0) {
					// ((mean - 1) * div) >> 18 in 32-bit pieces: div <= 2^18, so the product is below 2^50 and the result below 2^32
					const uint32_t m32 = (uint32_t)mean;
					const uint32_t m1 = m32 - 1;
					const uint32_t t = m32 < 2 ? 0u : __funnelshift_r(m1 * div, __umulhi(m1, div), 18);
					k = t ? 32u - (uint32_t)__clz((int)t) : 0u;
				}
				else {
					const unsigned long long t = ((mean - 1) * div) >> 18;
					k = t ? ilog2_u64(t) + 1 : 0u;
				}
				if(k > rice_cap) k = rice_cap;
				if(own) params_all[n] = (uint8_t)k;
				return own ? count_rice_bits(k, psamp, mean) : 0u;
			};
			auto close_order = [&](int po, unsigned long long lane_bits) {
				unsigned long long total;
				if(__any_sync(0xffffffffu, (lane_bits >> 27) != 0)) total = warp_sum_u64(lane_bits);
				else total = __reduce_add_sync(0xffffffffu, (unsigned)lane_bits);  // 32 lanes x 2^27 cannot wrap
				total += kEntropyTypeLen + kRiceOrderLen;
				const uint32_t bits = (uint32_t)(total < 0xffffffffull ? total : 0xffffffffull);
				if(best_r == 0 || bits < best_r) { best_r = bits; best_po = po; }
			};
			// orders >= 5: a lane owns 2^(po-5) consecutive nodes, merged in registers on the way down
			unsigned long long cur;  // after this block: the node of order `lev` this lane's group of 32 >> lev lanes stands for
			int lev;
			if(max_po >= 5) {
				unsigned long long v[8];
				const int cnt0 = 1 << (max_po - 5);
	#pragma unroll
				for(int i = 0; i < 8; i++) v[i] = i < cnt0 ? leaf[lane * cnt0 + i] : 0ull;
				int po = max_po;
	#pragma unroll 1
				for(; po >= 5 && po >= min_po; po--) {
					const int cnt = 1 << (po - 5);
					const uint32_t pbase = (uint32_t)(bs >> po);
					const uint32_t div_rest = 0x40000u / pbase, div_first = 0x40000u / (pbase - (uint32_t)order);
					unsigned long long b = 0;
	#pragma unroll
					for(int i = 0; i < 8; i++)
						if(i < cnt) {
							const int p = lane * cnt + i;
							b += node_bits(v[i], p == 0 ? pbase - (uint32_t)order : pbase, p == 0 ? div_first : div_rest, (1 << po) + p, true);
						}
					close_order(po, b);
	#pragma unroll
					for(int i = 0; i < 4; i++)
						if(2 * i + 1 < cnt) v[i] = v[2 * i] + v[2 * i + 1];
				}
				cur = v[0];
				lev = 5;
			}
			else {
				cur = leaf[lane >> (5 - max_po)];
				lev = max_po;
			}
			// orders <= 4 (31 nodes): heap node n = (1 << L) + p is evaluated once, by lane n - 1. Walking down, every lane of a
			// node's group holds the node's sum; the evaluating lane fetches it from the group's first lane.
			if(min_po <= 4) {
				const int n1 = lane + 1;
				const int myL = (int)ilog2_u32((uint32_t)n1);
				const int myP = n1 - (1 << myL);
				unsigned long long mine = 0;
	#pragma unroll 1
				for(int L = 4; L >= 0; L--) {
					if(L < lev) cur += __shfl_xor_sync(0xffffffffu, cur, 16 >> L);  // two order-(L+1) groups make one order-L group
					const unsigned long long got = __shfl_sync(0xffffffffu, cur, (myP << (5 - L)) & 31);
					if(myL == L) mine = got;
				}
				const int top = max_po < 4 ? max_po : 4;
				const bool active = lane < 31 && myL >= min_po && myL <= top;
				const uint32_t psamp = (uint32_t)(bs >> myL) - (myP == 0 ? (uint32_t)order : 0u);
				const uint32_t bits = node_bits(mine, psamp, 0x40000u / psamp, n1, active);
	#pragma unroll 1
				for(int L = top; L >= min_po; L--)
					if(true) close_order(L, (active && myL == L) ? bits : 0u);
			}

			uint32_t estimate = kSubframeHeaderBits + (uint32_t)wasted;
			if(type == SF_FIXED) estimate += (uint32_t)order * (uint32_t)sbps;
			else estimate += kQlpPrecisionLen + kQlpShiftLen + (uint32_t)order * (uint32_t)(precision + sbps);
			if(best_r < 0xffffffffu - estimate) estimate += best_r;
			else estimate = 0xffffffffu;
			const bool better = (type == SF_LPC ? estimate > 0 : true) && estimate < best_bits;
			if(better) {
				__syncwarp();  // params_all was written by the lanes that own the nodes
				uint32_t any15 = 0;
				for(int p = lane; p < (1 << best_po); p += 32) {
					const uint8_t k = params_all[(1 << best_po) + p];
					b_params[p] = k;
					any15 |= (k >= kRiceEscape) ? 1u : 0u;
				}
				any15 = warp_or(any15);
				best_bits = estimate;
				b_idx = cand_index;
				b_type = type; b_order = order; b_prec = precision; b_shift = shift; b_method = any15 ? 1 : 0; b_po = best_po; b_wide = wide;
	#pragma unroll
				for(int j = 0; j < MAXORD; j++) b_q[j] = (type == SF_LPC) ? q[j] : 0;
			}
			__syncwarp();
		};


		if(bs > (int)kMaxFixedOrder) {
			if(part == 0 || WPS == 2) {
				// fixed-predictor scan (fixed.c:222-290) + constant detection; the two warps of a signal take alternate tiles
				unsigned long long te[5] = {0, 0, 0, 0, 0};
				uint32_t diff = 0;
				const int32_t x0 = xs[0];
				// The order-k error is the k-th finite difference; in wrapping 32-bit arithmetic it equals the
				// reference's value whenever that fits an int32: |e4| <= 16 * 2^(sbps-1), i.e. sbps <= 27 (the
				// engine's scope is sbps <= 25). |e| sums: a lane adds bs/32 values below 2^(sbps+3) per order, so
				// 32-bit lane totals are exact when sbps + 3 + log2(bs/32) <= 32; otherwise they are flushed to
				// 64 bits every 4 samples (4 * 2^28 < 2^32).
				const bool lane_total_fits = (uint32_t)(sbps + 3) + ilog2_u32((uint32_t)(2 * (bs / 32) - 1)) <= 32u;
				uint32_t t32[5] = {0, 0, 0, 0, 0};
		#pragma unroll 1
				for(int t = (WPS == 2 ? part : 0); t < ntiles; t += WPS) {
					const int row = t * 32 + lane;
					int xw[4 + R_T];
					{
						const int4 *pv = reinterpret_cast<const int4 *>(xs + row * 36);
						const int4 hv = pv[-1 - GAPV];  // row 0 reads the zero row
						xw[0] = hv.x; xw[1] = hv.y; xw[2] = hv.z; xw[3] = hv.w;
		#pragma unroll
						for(int k = 0; k < R_T / 4; k++) {
							const int4 v = pv[k];
							xw[4 + 4 * k] = v.x; xw[5 + 4 * k] = v.y; xw[6 + 4 * k] = v.z; xw[7 + 4 * k] = v.w;
						}
					}
					// difference pyramid: e1[k] belongs to sample k-3, e2[k] to k-2, e3[k] to k-1, e4 to m
					int e1[R_T + 3], e2[R_T + 2], e3[R_T + 1];
		#pragma unroll
					for(int k = 0; k < R_T + 3; k++) e1[k] = xw[k + 1] - xw[k];
		#pragma unroll
					for(int k = 0; k < R_T + 2; k++) e2[k] = e1[k + 1] - e1[k];
		#pragma unroll
					for(int k = 0; k < R_T + 1; k++) e3[k] = e2[k + 1] - e2[k];
		#pragma unroll
					for(int m = 0; m < R_T; m++) {
						diff |= (uint32_t)(xw[4 + m] ^ x0);
						const bool counted = m >= (int)kMaxFixedOrder || row != 0;  // fixed.c:222-290 starts at sample 4
						if(counted) {
							t32[0] = __sad(xw[4 + m], 0, t32[0]);
							t32[1] = __sad(e1[m + 3], 0, t32[1]);
							t32[2] = __sad(e2[m + 2], 0, t32[2]);
							t32[3] = __sad(e3[m + 1], 0, t32[3]);
							t32[4] = __sad(e3[m + 1] - e3[m], 0, t32[4]);
						}
						if((m & 3) == 3 && !lane_total_fits) {
		#pragma unroll
							for(int k = 0; k < 5; k++) { te[k] += t32[k]; t32[k] = 0; }
						}
					}
				}
		#pragma unroll
				for(int k = 0; k < 5; k++) te[k] += t32[k];
				uint32_t eq = diff == 0 ? 1u : 0u;
		#pragma unroll
				for(int k = 0; k < 5; k++) te[k] = warp_sum_u64(te[k]);
				eq = warp_and(eq);
				if(WPS == 2) {
					// the second warp hands its partial sums to the first through shared memory (named barrier: 64 threads of the signal)
					unsigned long long *xch = xch_all + 6 * sidx;
					if(part == 1) {
						if(lane == 0) {
#pragma unroll
							for(int k = 0; k < 5; k++) xch[k] = te[k];
							xch[5] = eq;
						}
						__threadfence_block();
						asm volatile("bar.arrive %0, 64;" ::"r"(1 + sidx) : "memory");
					}
					else {
						asm volatile("bar.sync %0, 64;" ::"r"(1 + sidx) : "memory");
#pragma unroll
						for(int k = 0; k < 5; k++) te[k] += xch[k];
						eq &= (uint32_t)xch[5];
					}
				}
				if(part == 0) {
				int guess;
				{
					const unsigned long long m34 = te[3] < te[4] ? te[3] : te[4], m234 = te[2] < m34 ? te[2] : m34, m1234 = te[1] < m234 ? te[1] : m234;
					if(te[0] <= m1234) guess = 0;
					else if(te[1] <= m234) guess = 1;
					else if(te[2] <= m34) guess = 2;
					else if(te[3] <= te[4]) guess = 3;
					else guess = 4;
				}
				float rbps[5];
				{
					// one lane per order evaluates the log (fixed.c:284-288); the results are broadcast
					const double n = (double)(uint32_t)(bs - (int)kMaxFixedOrder);
					unsigned long long mine = te[0];
		#pragma unroll
					for(int k = 1; k < 5; k++) mine = lane == k ? te[k] : mine;
					const float r = (float)((mine > 0) ? fb_log(M_LN2 * (double)mine / n) / M_LN2 : 0.0);
		#pragma unroll
					for(int k = 0; k < 5; k++) rbps[k] = __shfl_sync(0xffffffffu, r, k);
				}
				is_constant = !P.dis_const && rbps[1] == 0.0f && eq;
				if(is_constant) {
					const uint32_t cbits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)sbps;
					if(cbits < best_bits) { best_bits = cbits; b_type = SF_CONSTANT; b_idx = 0; }
				}
				else if(!P.dis_fixed || (P.max_order == 0 && best_bits == 0xffffffffu)) {
					int lo, hi;
					if(P.exhaustive) { lo = 0; hi = (int)kMaxFixedOrder; }
					else lo = hi = guess;
					if(hi >= bs) hi = bs - 1;
					for(int fo = lo; fo <= hi; fo++) {
						if(rbps[fo] >= (float)sbps) continue;
						int q[MAXORD];
#pragma unroll
						for(int j = 0; j < MAXORD; j++) q[j] = fixed_tap(fo, j);
						evaluate(fo, SF_FIXED, fo, 0, 0, 0, 0, q);
					}
				}
				}  // part == 0
			}
			if(P.max_order > 0 && !is_constant) {
				// LPC candidates: a queue per signal; a constant signal's LPC results (second warp) are dropped at the merge
				const CandDesc *cd = cdesc + ((size_t)blk * P.nsig + sig0 + sidx) * P.nslots;
				for(;;) {
					int c = 0;
					if(lane == 0) c = atomicAdd(&queues[sidx], 1);
					c = __shfl_sync(0xffffffffu, c, 0);
					if(c >= P.nslots) break;
					const CandDesc *D = cd + c;
					if(!__ldg(&D->valid)) continue;
					int q[MAXORD];
#pragma unroll
					for(int j = 0; j < MAXORD; j++) q[j] = __ldg(&D->qlp[j]);
					evaluate(5 + c, SF_LPC, __ldg(&D->order), __ldg(&D->precision), __ldg(&D->shift), __ldg(&D->wide), __ldg(&D->limit), q);
				}
			}
		}
	}

	// ---- merge the warps of a signal, write the plan
	if(WPS > 1 && active && part != 0 && lane == 0) {
		SearchResult5 &Rz = results[sidx];
		Rz.best_bits = best_bits; Rz.idx = b_idx; Rz.type = b_type; Rz.order = b_order; Rz.prec = b_prec; Rz.shift = b_shift;
		Rz.method = b_method; Rz.po = b_po; Rz.wide = b_wide;
#pragma unroll
		for(int j = 0; j < MAXORD; j++) Rz.q[j] = b_q[j];
	}
	__syncthreads();
	if(!have_signal || part != 0 || skip_sig) return;
	SubframePlan *plan = plans + (size_t)blk * P.nsig + sig0 + sidx;
	if(!active) {
		if(lane == 0) { plan->type = -1; plan->est_bits = 0xffffffffu; }
		return;
	}
	const uint8_t *win_params = b_params;
	if(WPS > 1 && !is_constant) {
		const SearchResult5 &Rz = results[sidx];
		const bool other = Rz.best_bits < best_bits || (Rz.best_bits == best_bits && Rz.idx >= 0 && (b_idx < 0 ? false : Rz.idx < b_idx));
		if(other) {
			best_bits = Rz.best_bits; b_type = Rz.type; b_order = Rz.order; b_prec = Rz.prec; b_shift = Rz.shift; b_method = Rz.method; b_po = Rz.po; b_wide = Rz.wide;
#pragma unroll
			for(int j = 0; j < MAXORD; j++) b_q[j] = Rz.q[j];
			win_params = scratch0 + (size_t)(warp + 1) * scratch_bytes + ((size_t)8 << P.max_po) + ((size_t)2 << P.max_po);
		}
	}
	if(best_bits == 0xffffffffu) {  // nothing was allowed to win: verbatim after all (stream_encoder.c:4281-4284)
		b_type = SF_VERBATIM;
		best_bits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)bs * (uint32_t)sbps;
	}
	if(lane == 0) {
		plan->type = b_type; plan->order = b_order; plan->wasted = wasted; plan->bps = sbps;
		plan->precision = b_prec; plan->shift = b_shift; plan->method = b_method; plan->porder = b_po;
		plan->est_bits = best_bits; plan->wide = b_wide;
#pragma unroll
		for(int j = 0; j < FB200_MAX_LPC_ORDER; j++) plan->qlp[j] = (j < MAXORD) ? b_q[j < MAXORD ? j : 0] : 0;
	}
	for(int p = lane; p < kMaxPartitions; p += 32) plan->params[p] = p < (1 << P.max_po) ? win_params[p] : 0;
}

}  // namespace fb200
