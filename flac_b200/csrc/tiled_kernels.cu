// tiled_kernels.cu -- stage B for frames that do not fit one CTA's shared memory: k_search_tiled, k_emit_tiled, k_join_tiled.
//
// k_search keeps a whole signal and its residual in shared memory, k_emit a whole frame; that bounds the blocksize x channels
// x bits they take on a device. These kernels stream a signal through shared memory in tiles of kTileN samples, each with
// the kTileHist samples in front of it as predictor history (1-D TMA bulk copies onto a two-slot mbarrier ring), and keep
// nothing else of the signal resident: the search holds per-partition |residual| sums of a group of candidates, the emit
// packs each subframe into a staging region in global memory, and the join splices a frame's subframes behind its header.
// Every decision rule and every bit is k_search's / k_emit's; the frames go to d_slots for the unchanged k_scan + k_gather.
#include "device_common.cuh"

namespace fb200 {

constexpr int kTileN = 2048;                    // samples per tile (a multiple of 4: bulk copies move whole 16-byte units)
constexpr int kTileHist = FB200_MAX_LPC_ORDER;  // history in front of a tile: the largest predictor order
constexpr int kTileStride = kTileHist + kTileN;
constexpr size_t kRingBytes = 2 * kTileStride * sizeof(int32_t);
constexpr int kTiledThreads = 256;
constexpr int kTiledWarps = kTiledThreads / 32;
constexpr int kTiledGroup = 16;                 // candidates evaluated by one pass over the signal
constexpr int kJoinThreads = 512;

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// Streams g[0 .. bs) through the ring: body(start, n, x) sees samples start .. start+n-1 as x[0 .. n) and the kTileHist
// samples in front of them as x[-kTileHist .. 0) (undefined in the first tile, where no predictor reaches back that far).
// The copy of tile t+1 is in flight while tile t is processed. seq counts the tiles the ring has carried (slot seq & 1, phase
// (seq >> 1) & 1) and is the same in every thread; every thread calls this. The copies read whole 16-byte units: up to 3
// samples past bs, inside the signal's bs_stride row.
template <class F>
__device__ __forceinline__ void stream_tiles(const int32_t *g, int bs, int32_t *ring, uint64_t *bars, unsigned &seq, F &&body)
{
	const int ntiles = (bs + kTileN - 1) / kTileN;
	auto issue = [&](int t) {
		if(threadIdx.x == 0 && t < ntiles) {
			const unsigned slot = (seq + (unsigned)t) & 1u;
			const int start = t * kTileN, n4 = (min(kTileN, bs - start) + 3) & ~3, h = t ? kTileHist : 0;
			fence_proxy_async_smem();  // the slot was last read through the generic proxy
			mbar_expect_tx(&bars[slot], (unsigned)(n4 + h) * 4u);
			tma_bulk_g2s(ring + slot * kTileStride + kTileHist - h, g + start - h, (unsigned)(n4 + h) * 4u, &bars[slot]);
		}
	};
	issue(0);
	for(int t = 0; t < ntiles; t++) {
		issue(t + 1);  // into the slot of tile t-1: every thread passed the barrier behind it
		const unsigned u = seq + (unsigned)t;
		mbar_wait(&bars[u & 1u], (u >> 1) & 1u);
		body(t * kTileN, min(kTileN, bs - t * kTileN), ring + (u & 1u) * kTileStride + kTileHist);
		__syncthreads();
	}
	seq += (unsigned)ntiles;
}

// Residual of sample x[0] (x[-1 .. -order] in front of it), with k_search's / k_emit's arithmetic: 32-bit fixed predictors
// (fixed.c:470-530), 32-bit LPC unless `wide`, else 64-bit (lpc.c:321-938). The caller narrows it to 32 bits.
__device__ __forceinline__ int64_t tiled_residual(int type, int order, const int *qlp, int shift, int wide, const int32_t *x)
{
	if(type == SF_FIXED) {
		int32_t r;
		switch(order) {
			case 0: r = x[0]; break;
			case 1: r = x[0] - x[-1]; break;
			case 2: r = x[0] - 2 * x[-1] + x[-2]; break;
			case 3: r = x[0] - 3 * x[-1] + 3 * x[-2] - x[-3]; break;
			default: r = x[0] - 4 * x[-1] + 6 * x[-2] - 4 * x[-3] + x[-4]; break;
		}
		return r;
	}
	if(!wide) {
		int32_t sum = 0;
		for(int j = 0; j < order; j++) sum += qlp[j] * x[-1 - j];
		return (int32_t)(x[0] - (sum >> shift));
	}
	int64_t sum = 0;
	for(int j = 0; j < order; j++) sum += (int64_t)qlp[j] * (int64_t)x[-1 - j];
	return (int64_t)x[0] - (sum >> shift);
}

// ================================================================ k_search_tiled
// One CTA per (block, signal). Pass 1 streams the signal once for the fixed-order abs sums and the constant test; then the
// candidates (fixed orders, then the LPC slots, in k_search's evaluation order) are evaluated kTiledGroup at a time: one
// pass over the tiles adds every candidate's |residual| into its partition sums at its own largest usable order, warps
// owning (candidate, slice of the tile) pairs; then a warp per candidate runs the partition-order search. The best is the
// first minimum over (estimate, candidate index) -- k_search's strict '<' in evaluation order.
struct TiledCand {
	int type, order, precision, shift, wide, limit;
	int max_po, min_po, psize, fail, po, method;
	uint32_t est;
	int qlp[FB200_MAX_LPC_ORDER];
};

struct TiledSearchShared {
	uint64_t bars[2];
	unsigned long long te[5];
	int all_equal, ncand, next, win;
	int cidx[kTiledGroup];
	TiledCand cand[kTiledGroup];
	uint32_t best_bits;
	int b_type, b_order, b_prec, b_shift, b_method, b_po, b_wide;
	int b_qlp[FB200_MAX_LPC_ORDER];
	uint8_t b_params[kMaxPartitions];
};

// dynamic shared memory: the ring, the group's partition sums and chosen parameters, per-warp search scratch
constexpr size_t kTsSums = kRingBytes;
constexpr size_t kTsParams = kTsSums + (size_t)kTiledGroup * kMaxPartitions * 8;
constexpr size_t kTsWtmp = kTsParams + (size_t)kTiledGroup * kMaxPartitions;
constexpr size_t kTsWparams = kTsWtmp + (size_t)kTiledWarps * (kMaxPartitions / 2) * 8;
constexpr size_t kSearchTiledSmem = kTsWparams + (size_t)kTiledWarps * 2 * kMaxPartitions;

__global__ void __launch_bounds__(kTiledThreads) k_search_tiled(EncK P, const int32_t *__restrict__ sig, const SigMeta *__restrict__ meta,
                                                               const CandDesc *__restrict__ cdesc, SubframePlan *__restrict__ plans)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ TiledSearchShared S;
	const int item = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, bs = P.bs;
	if(P.redo) {
		const int blk = item / P.nsig;
		if(!P.redo[blk] || item - blk * P.nsig < P.channels - 1) return;
	}
	const SigMeta M = meta[item];
	SubframePlan *plan = plans + item;
	if(M.bps == 0) {
		if(tid == 0) { plan->type = -1; plan->est_bits = 0xffffffffu; }
		return;
	}
	int32_t *ring = reinterpret_cast<int32_t *>(smem_raw);
	unsigned long long *sums = reinterpret_cast<unsigned long long *>(smem_raw + kTsSums);
	uint8_t *cparams = smem_raw + kTsParams;
	unsigned long long *wtmp = reinterpret_cast<unsigned long long *>(smem_raw + kTsWtmp) + warp * (kMaxPartitions / 2);
	uint8_t *wparams = smem_raw + kTsWparams + warp * 2 * kMaxPartitions;
	const int sbps = M.bps, wasted = M.wasted;
	const int32_t *g = sig + (size_t)item * P.bs_stride;

	if(tid == 0) {
		mbar_init(&S.bars[0], 1);
		mbar_init(&S.bars[1], 1);
		mbar_fence_init();
		S.all_equal = 1;
		// verbatim baseline (evaluate_verbatim_subframe_, :4669-4699; :4082-4086)
		S.b_type = SF_VERBATIM; S.b_order = 0; S.b_prec = 0; S.b_shift = 0; S.b_method = 0; S.b_po = 0; S.b_wide = 0;
		if(P.dis_verb && bs >= (int)kMaxFixedOrder) S.best_bits = 0xffffffffu;
		else S.best_bits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)bs * (uint32_t)sbps;
	}
	if(tid < 5) S.te[tid] = 0;
	if(tid < FB200_MAX_LPC_ORDER) S.b_qlp[tid] = 0;
	for(int p = tid; p < kMaxPartitions; p += kTiledThreads) S.b_params[p] = 0;
	__syncthreads();
	unsigned seq = 0;

	if(bs > (int)kMaxFixedOrder) {
		// ---- pass 1: fixed.c:222-290 abs sums of the 0..4th differences over samples 4..bs-1, and the all-equal test
		unsigned long long te[5] = {0, 0, 0, 0, 0};
		uint32_t eq = 1;
		const int32_t x0 = g[0];
		stream_tiles(g, bs, ring, S.bars, seq, [&](int start, int n, const int32_t *x) {
			for(int j = tid; j < n; j += kTiledThreads) {
				const int i = start + j;
				if(i >= 1) eq &= (x[j] == x0) ? 1u : 0u;
				if(i >= (int)kMaxFixedOrder) {
					const int64_t d0 = x[j], d1 = x[j - 1], d2 = x[j - 2], d3 = x[j - 3], d4 = x[j - 4];
					const int64_t e1 = d0 - d1, e2 = d0 - 2 * d1 + d2, e3 = d0 - 3 * d1 + 3 * d2 - d3, e4 = d0 - 4 * d1 + 6 * d2 - 4 * d3 + d4;
					te[0] += (unsigned long long)(d0 < 0 ? -d0 : d0);
					te[1] += (unsigned long long)(e1 < 0 ? -e1 : e1);
					te[2] += (unsigned long long)(e2 < 0 ? -e2 : e2);
					te[3] += (unsigned long long)(e3 < 0 ? -e3 : e3);
					te[4] += (unsigned long long)(e4 < 0 ? -e4 : e4);
				}
			}
		});
#pragma unroll
		for(int k = 0; k < 5; k++) {
			te[k] = warp_sum_u64(te[k]);
			if(lane == 0) atomicAdd(&S.te[k], te[k]);
		}
		eq = warp_and(eq);
		if(lane == 0 && !eq) S.all_equal = 0;
		__syncthreads();
		if(fixed_guess_avx2(P, bs, sbps)) {
			if(tid == 0) fixed_guess_avx2_fixup(g, bs, S.te);  // from global memory: the positions lie anywhere in the signal
			__syncthreads();
		}
		const unsigned long long tt[5] = {S.te[0], S.te[1], S.te[2], S.te[3], S.te[4]};
		float rbps[5];
		const int guess = fixed_best_order(tt, bs, rbps);
		const bool is_constant = !P.dis_const && rbps[1] == 0.0f && S.all_equal != 0;  // stream_encoder.c:4111-4140
		if(is_constant) {
			if(tid == 0) {
				const uint32_t cbits = kSubframeHeaderBits + (uint32_t)wasted + (uint32_t)sbps;  // :4466-4487
				if(cbits < S.best_bits) { S.best_bits = cbits; S.b_type = SF_CONSTANT; }
			}
			__syncthreads();
		}
		else {
			int flo = 0, fhi = -1;
			if(!P.dis_fixed || (P.max_order == 0 && S.best_bits == 0xffffffffu)) {
				if(P.exhaustive) { flo = 0; fhi = (int)kMaxFixedOrder; }
				else flo = fhi = guess;
				if(fhi >= bs) fhi = bs - 1;
			}
			const int nfix = fhi - flo + 1, nall = nfix + (P.max_order > 0 ? P.nslots : 0);
			uint32_t fixlive = 0;  // bit k: fixed order k is tried (:4166)
#pragma unroll
			for(int k = 0; k < 5; k++)
				if(!(rbps[k] >= (float)sbps)) fixlive |= 1u << k;
			const CandDesc *cd = cdesc + (size_t)item * P.nslots;
			int v = 0;  // next candidate in evaluation order: fixed orders flo..fhi (:4166 skips), then the valid LPC slots
			while(v < nall) {
				// ---- the next group: warp 0 compacts the live candidates 32 at a time
				if(warp == 0) {
					int n = 0;
					while(v < nall && n < kTiledGroup) {
						const int vv = v + lane;
						bool live = false;
						if(vv < nall) live = vv < nfix ? ((fixlive >> (flo + vv)) & 1u) != 0 : cd[vv - nfix].valid != 0;
						const uint32_t m = __ballot_sync(0xffffffffu, live);
						const int rank = __popc(m & ((1u << lane) - 1u)), take = min(__popc(m), kTiledGroup - n);
						if(live && rank < take) S.cidx[n + rank] = vv;
						const uint32_t lastm = __ballot_sync(0xffffffffu, live && rank == take - 1);
						v += (take < __popc(m)) ? __ffs((int)lastm) : min(32, nall - v);
						n += take;
					}
					if(lane == 0) { S.ncand = n; S.next = v; }
				}
				__syncthreads();
				v = S.next;
				const int ng = S.ncand;
				if(ng == 0) break;  // no live candidate left (v == nall)
				for(int c = warp; c < ng; c += kTiledWarps) {
					TiledCand &C = S.cand[c];
					const int vv = S.cidx[c];
					if(vv < nfix) {
						if(lane == 0) { C.type = SF_FIXED; C.order = flo + vv; C.precision = 0; C.shift = 0; C.wide = 0; C.limit = 0; }
						C.qlp[lane] = 0;
					}
					else {
						const CandDesc *D = cd + (vv - nfix);
						if(lane == 0) { C.type = SF_LPC; C.order = D->order; C.precision = D->precision; C.shift = D->shift; C.wide = D->wide; C.limit = D->limit; }
						C.qlp[lane] = D->qlp[lane];
					}
					__syncwarp();
					if(lane == 0) {
						// partition sums at the largest usable order (stream_encoder.c:4797-4835, format.c:550-562)
						int max_po = P.max_po;
						while(max_po > 0 && (bs >> max_po) <= C.order) max_po--;
						C.max_po = max_po; C.min_po = min(P.min_po, max_po); C.psize = bs >> max_po; C.fail = 0;
					}
					for(int p = lane; p < kMaxPartitions; p += 32) sums[c * kMaxPartitions + p] = 0;
				}
				__syncthreads();

				// ---- one pass over the tiles: warp w owns (candidate, slice) pairs and adds |residual| into the partition sums
				const int slices = ng >= kTiledWarps ? 1 : kTiledWarps / ng;
				stream_tiles(g, bs, ring, S.bars, seq, [&](int start, int n, const int32_t *x) {
					for(int w = warp; w < ng * slices; w += kTiledWarps) {
						const int c = w / slices, s = w - c * slices;
						const TiledCand &C = S.cand[c];
						const int type = C.type, order = C.order, shift = C.shift, wide = C.wide, limit = C.limit, psize = C.psize;
						int j0 = (n * s) / slices;
						const int j1 = (n * (s + 1)) / slices;
						if(start + j0 < order) j0 = order - start;  // warm-up samples have no residual
						unsigned long long *cs = sums + c * kMaxPartitions;
						int curp = 0, pend = -1;
						unsigned long long acc = 0;
						bool bad = false;
						for(int j = j0 + lane; j < j1; j += 32) {
							const int i = start + j;
							const int64_t r = tiled_residual(type, order, C.qlp, shift, wide, x + j);
							if(wide && limit && (r <= (int64_t)INT32_MIN || r > (int64_t)INT32_MAX)) bad = true;  // lpc.c:868-884
							if(i >= pend) {
								if(acc) atomicAdd(&cs[curp], acc);
								acc = 0;
								curp = i / psize;
								pend = (curp + 1) * psize;
							}
							acc += abs_u32((int32_t)r);
						}
						if(acc) atomicAdd(&cs[curp], acc);
						if(bad) S.cand[c].fail = 1;
					}
				});

				// ---- a warp per candidate: partition order / Rice parameter search and the estimate
				for(int c = warp; c < ng; c += kTiledWarps) {
					TiledCand &C = S.cand[c];
					if(C.fail) continue;  // rejected (evaluate_lpc_subframe_ returns 0, stream_encoder.c:4601-4609)
					unsigned long long *cs = sums + c * kMaxPartitions;
					const int order = C.order, nparts_max = 1 << C.max_po;
					const bool narrow = (uint32_t)(sbps + (int)kMaxExtraResidualBps) < 32u - ilog2_u32((uint32_t)C.psize);
					if(narrow)
						for(int p = lane; p < nparts_max; p += 32) cs[p] = (unsigned long long)(uint32_t)cs[p];
					__syncwarp();
					int best_po;
					const uint32_t best_r = rice_search_warp(P, bs, order, C.max_po, C.min_po, cs, wtmp, wparams, &best_po);
					__syncwarp();
					// estimate (evaluate_fixed_subframe_ :4550-4554, evaluate_lpc_subframe_ :4655-4659)
					uint32_t estimate = kSubframeHeaderBits + (uint32_t)wasted;
					if(C.type == SF_FIXED) estimate += (uint32_t)order * (uint32_t)sbps;
					else estimate += kQlpPrecisionLen + kQlpShiftLen + (uint32_t)order * (uint32_t)(C.precision + sbps);
					if(best_r < 0xffffffffu - estimate) estimate += best_r;
					else estimate = 0xffffffffu;
					uint32_t any15 = 0;
					for(int p = lane; p < (1 << best_po); p += 32) {
						const uint8_t k = wparams[(1 << best_po) - 1 + p];
						cparams[c * kMaxPartitions + p] = k;
						any15 |= (k >= kRiceEscape) ? 1u : 0u;
					}
					any15 = warp_or(any15);
					if(lane == 0) { C.est = estimate; C.po = best_po; C.method = any15 ? 1 : 0; }  // RICE2 when a parameter needs 5 bits (:4786-4791)
					__syncwarp();
				}
				__syncthreads();

				// ---- merge in evaluation order (strict '<', stream_encoder.c:4191-4194, 4265-4269)
				if(tid == 0) {
					int win = -1;
					for(int c = 0; c < ng; c++) {
						const TiledCand &C = S.cand[c];
						if(C.fail) continue;
						if((C.type == SF_LPC ? C.est > 0 : true) && C.est < S.best_bits) { S.best_bits = C.est; win = c; }
					}
					S.win = win;
				}
				__syncthreads();
				const int win = S.win;
				if(win >= 0) {
					const TiledCand &C = S.cand[win];
					if(tid == 0) { S.b_type = C.type; S.b_order = C.order; S.b_prec = C.precision; S.b_shift = C.shift; S.b_method = C.method; S.b_po = C.po; S.b_wide = C.wide; }
					if(tid < FB200_MAX_LPC_ORDER) S.b_qlp[tid] = (C.type == SF_LPC && tid < C.order) ? C.qlp[tid] : 0;
					for(int p = tid; p < (1 << C.po); p += kTiledThreads) S.b_params[p] = cparams[win * kMaxPartitions + p];
				}
				__syncthreads();
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
	for(int p = tid; p < kMaxPartitions; p += kTiledThreads) plan->params[p] = S.b_params[p];
}

// ================================================================ k_emit_tiled
// One CTA per (block, channel): the subframe's header, then its residual (or verbatim samples) tile by tile with k_emit's
// arithmetic, packed MSB first with BitPut into the subframe's zeroed staging region in global memory. Within a tile every
// thread packs a run of samples at the offset a block scan of the run lengths gives it; the offset carries from tile to tile.
// stage_bits receives the subframe's exact bit count, or 0xffffffff when it would exceed cap_bits.
__global__ void __launch_bounds__(kTiledThreads) k_emit_tiled(EncK P, const int32_t *__restrict__ sig, const int *__restrict__ blkflags,
                                                             const SubframePlan *__restrict__ plans, uint32_t *__restrict__ stage,
                                                             uint32_t *__restrict__ stage_bits, int sub_words, uint32_t cap_bits)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2];
	__shared__ uint32_t s_warp[9];
	__shared__ int s_qlp[FB200_MAX_LPC_ORDER];
	__shared__ int32_t s_res[kTileN];
	const int blk = blockIdx.x / P.channels, c = blockIdx.x - blk * P.channels, tid = threadIdx.x, bs = P.bs;
	int32_t *ring = reinterpret_cast<int32_t *>(smem_raw);
	const SubframePlan *bp = plans + (size_t)blk * P.nsig;
	const int sidx = subframe_signal(P, channel_assignment(P, bp, blkflags[blk]), c);
	const SubframePlan *pl = bp + sidx;
	const int type = pl->type, order = pl->order, sbps = pl->bps, shift = pl->shift, wide = pl->wide;
	const int32_t *g = sig + ((size_t)blk * P.nsig + sidx) * P.bs_stride;
	uint32_t *words = stage + (size_t)blockIdx.x * sub_words;
	const uint32_t hbits = subframe_header_bits(pl);

	for(uint32_t w = tid; w <= (hbits >> 5); w += kTiledThreads) words[w] = 0;
	if(tid < FB200_MAX_LPC_ORDER) s_qlp[tid] = pl->qlp[tid];
	if(tid == 0) {
		mbar_init(&bars[0], 1);
		mbar_init(&bars[1], 1);
		mbar_fence_init();
	}
	__syncthreads();
	if(tid == 0) put_subframe_header(words, 0, pl, g);
	uint32_t base = hbits;
	bool over = false;
	if(type == SF_VERBATIM || type == SF_FIXED || type == SF_LPC) {
		const int psize = bs >> pl->porder;
		const uint32_t plen = pl->method ? kRice2ParamLen : kRiceParamLen;
		unsigned seq = 0;
		stream_tiles(g, bs, ring, bars, seq, [&](int start, int n, const int32_t *x) {
			if(over) return;
			if(type == SF_VERBATIM) {
				// n raw samples of sbps bits: fixed width, no scan
				const uint32_t b0 = base + (uint32_t)start * (uint32_t)sbps, b1 = b0 + (uint32_t)n * (uint32_t)sbps;
				if(b1 > cap_bits) { over = true; return; }
				for(uint32_t w = (b0 >> 5) + 1 + tid; w <= (b1 >> 5); w += kTiledThreads) words[w] = 0;
				__syncthreads();
				const int R = (n + kTiledThreads - 1) / kTiledThreads;
				const int j0 = tid * R, j1 = min(n, j0 + R);
				if(j0 < j1) {
					BitPut bw;
					bw.init(words, b0 + (uint32_t)j0 * (uint32_t)sbps);
					for(int j = j0; j < j1; j++) bw.put(mask_bits(x[j], (uint32_t)sbps), (uint32_t)sbps);
					bw.finish();
				}
				return;
			}
			// residual of the tile (same arithmetic as k_emit)
			const int jlo = max(0, order - start);
			for(int j = jlo + tid; j < n; j += kTiledThreads) s_res[j] = (int32_t)tiled_residual(type, order, s_qlp, shift, wide, x + j);
			__syncthreads();
			// partitioned Rice coding (stream_encoder_framing.c:538-594, bitwriter.c:575-706)
			const int R = (n - jlo + kTiledThreads - 1) / kTiledThreads;
			const int i0 = start + jlo + tid * R, i1 = min(start + n, i0 + R);
			uint32_t mybits = 0;
			if(i0 < i1) {
				int p = i0 / psize;
				int next = (p + 1) * psize;
				uint32_t k = __ldg(&pl->params[p]);
				for(int i = i0; i < i1; i++) {
					if(i == next) { p++; next += psize; k = __ldg(&pl->params[p]); }
					if(i == p * psize || i == order) mybits += plen;
					const int32_t r = s_res[i - start];
					const uint32_t u = ((uint32_t)r << 1) ^ (uint32_t)(r >> 31);
					mybits += (u >> k) + 1 + k;
				}
			}
			uint32_t total;
			const uint32_t off = block_exclusive_scan_256(mybits, s_warp, &total);
			if(base + total > cap_bits || base + total < base) { over = true; return; }
			for(uint32_t w = (base >> 5) + 1 + tid; w <= ((base + total) >> 5); w += kTiledThreads) words[w] = 0;
			__syncthreads();
			if(i0 < i1) {
				BitPut bw;
				bw.init(words, base + off);
				int p = i0 / psize;
				int next = (p + 1) * psize;
				uint32_t k = __ldg(&pl->params[p]);
				for(int i = i0; i < i1; i++) {
					if(i == next) { p++; next += psize; k = __ldg(&pl->params[p]); }
					if(i == p * psize || i == order) bw.put(k, plen);
					const int32_t r = s_res[i - start];
					const uint32_t u = ((uint32_t)r << 1) ^ (uint32_t)(r >> 31);
					bw.skip(u >> k);
					bw.put((1u << k) | (u & ((1u << k) - 1u)), k + 1);
				}
				bw.finish();
			}
			base += total;
		});
		if(type == SF_VERBATIM) base = hbits + (uint32_t)bs * (uint32_t)sbps;
	}
	if(tid == 0) stage_bits[blockIdx.x] = over ? 0xffffffffu : base;
}

// ================================================================ k_join_tiled
// One CTA per frame: the frame header + CRC-8 (k_emit's), then the subframes spliced in behind it with funnel shifts,
// streamed from the staging regions (L2) straight into the frame's d_slots slot. Every thread assembles a contiguous run of
// output words and takes the CRC-16 of its bytes on the way; the runs' CRCs combine over GF(2) (crc(A.B) = crc(A) x^8|B|
// + crc(B)). Zero padding to a byte boundary, the CRC-16, and the frame size in frame_bytes for k_scan / k_gather.
__global__ void __launch_bounds__(kJoinThreads) k_join_tiled(EncK P, const int *__restrict__ blkflags, const SubframePlan *__restrict__ plans,
                                                            const uint32_t *__restrict__ stage, const uint32_t *__restrict__ stage_bits, int sub_words,
                                                            uint8_t *__restrict__ slots, uint32_t *__restrict__ frame_bytes,
                                                            uint32_t *__restrict__ chan_assign_out, int *__restrict__ err)
{
	__shared__ uint16_t s_crctab[256];
	__shared__ uint32_t s_hdr[5];
	__shared__ uint32_t s_off[FB200_MAX_CHANNELS], s_len[FB200_MAX_CHANNELS];
	__shared__ uint32_t s_part[kJoinThreads / 32];
	__shared__ uint32_t s_total;
	__shared__ int s_ca, s_bad;
	const int blk = blockIdx.x, tid = threadIdx.x, ch = P.channels;
	if(tid < 256) s_crctab[tid] = (uint16_t)crc16_entry((uint32_t)tid);
	if(tid < 5) s_hdr[tid] = 0;
	__syncthreads();
	if(tid == 0) {
		const int ca = channel_assignment(P, plans + (size_t)blk * P.nsig, blkflags[blk]);
		const uint32_t frame_number = frame_number_of(P, blk);
		const FrameHdr H = frame_header_layout(P.bs, P.sample_rate, frame_number);
		put_frame_header(P, s_hdr, P.bs, frame_number, ca, H);
		uint32_t off = H.bits;
		int bad = 0;
		for(int c = 0; c < ch; c++) {
			const uint32_t len = stage_bits[(size_t)blk * ch + c];
			bad |= len == 0xffffffffu;
			s_off[c] = off;
			s_len[c] = len;
			off += len;
		}
		s_total = off; s_ca = ca; s_bad = bad;
	}
	__syncthreads();
	if(s_bad) {
		if(tid == 0) { atomicExch(err, 2); frame_bytes[blk] = 0; }
		return;
	}
	const uint32_t total = s_total, nbytes = (total + 7) >> 3, nwords = (nbytes + 3) >> 2;
	const uint32_t per = (nwords + kJoinThreads - 1) / kJoinThreads;
	const uint32_t w0 = min(nwords, (uint32_t)tid * per), w1 = min(nwords, w0 + per);
	uint8_t *fb = slots + (size_t)blk * P.slot_stride;
	uint32_t *dst = reinterpret_cast<uint32_t *>(fb);
	const uint32_t *sub = stage + (size_t)blk * ch * sub_words;
	uint32_t crc = 0;
	for(uint32_t w = w0; w < w1; w++) {
		uint32_t v = w < 5 ? s_hdr[w] : 0u;  // s_hdr is zero behind the header
		const uint32_t lo_bit = 32u * w;
		for(int c = 0; c < ch; c++) {
			const uint32_t s = s_off[c], L = s_len[c];
			if(lo_bit + 32u <= s || lo_bit >= s + L) continue;
			const uint32_t *W = sub + (size_t)c * sub_words;
			if(lo_bit >= s) {
				// a region is zero behind its last bit; the word after its last word is never read
				const uint32_t b = lo_bit - s, q = b >> 5;
				v |= __funnelshift_l(32u * (q + 1) < L ? W[q + 1] : 0u, W[q], b & 31u);
			}
			else v |= W[0] >> (s - lo_bit);
		}
		dst[w] = __byte_perm(v, 0, 0x0123);
		const uint32_t nb = min(4u, nbytes - 4u * w);
		for(uint32_t k = 0; k < nb; k++) {
			const uint32_t byte = (v >> (24 - 8 * k)) & 0xffu;
			crc = ((crc << 8) & 0xffffu) ^ s_crctab[((crc >> 8) ^ byte) & 0xffu];
		}
	}
	{
		// shift this run's CRC past the bytes behind it: x^(8 * behind) mod the CRC-16 polynomial, square and multiply
		const uint32_t m = gf16_xpow(8u * (nbytes - min(nbytes, 4u * w1)));
		crc = gf16_mul(crc, m);
	}
	crc = __reduce_xor_sync(0xffffffffu, crc);
	if((tid & 31) == 0) s_part[tid >> 5] = crc;
	__syncthreads();
	if(tid == 0) {
		uint32_t f = 0;
		for(int i = 0; i < kJoinThreads / 32; i++) f ^= s_part[i];
		fb[nbytes] = (uint8_t)(f >> 8);
		fb[nbytes + 1] = (uint8_t)f;
		frame_bytes[blk] = nbytes + 2;
		if(chan_assign_out) chan_assign_out[blk] = (uint32_t)s_ca;
	}
}

size_t search_tiled_smem() { return kSearchTiledSmem; }

void launch_search_tiled(const EncK &k, const int32_t *sig, const SigMeta *meta, const CandDesc *cdesc, SubframePlan *plans, int nitems, cudaStream_t st)
{
	k_search_tiled<<<nitems, kTiledThreads, kSearchTiledSmem, st>>>(k, sig, meta, cdesc, plans);
}

void launch_emit_tiled(const EncK &k, const int32_t *sig, const int *blkflags, const SubframePlan *plans, uint32_t *stage, uint32_t *stage_bits,
                       int sub_words, uint32_t cap_bits, uint8_t *slots, uint32_t *frame_bytes, uint32_t *chan_assign, int *err, int nb, cudaStream_t st)
{
	k_emit_tiled<<<nb * k.channels, kTiledThreads, kRingBytes, st>>>(k, sig, blkflags, plans, stage, stage_bits, sub_words, cap_bits);
	k_join_tiled<<<nb, kJoinThreads, 0, st>>>(k, blkflags, plans, stage, stage_bits, sub_words, slots, frame_bytes, chan_assign, err);
}

void tiled_init(int device)
{
	(void)device;
	cudaFuncSetAttribute(k_search_tiled, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSearchTiledSmem);
}

}  // namespace fb200
