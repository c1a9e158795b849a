// general_kernels.cu -- the general kernels (any blocksize / channel count) and their launchers.
#include "encode_kernels.cuh"

namespace fb200 {

void launch_prep(const EncK &k, const int32_t *pcm, int32_t *sig, SigMeta *meta, int *blkflags, int nb, cudaStream_t st)
{
	k_prep<true><<<nb, 256, 0, st>>>(k, pcm, sig, meta, blkflags);
}

void launch_meta(const EncK &k, const int32_t *pcm, SigMeta *meta, int *blkflags, int nb, cudaStream_t st)
{
	k_prep<false><<<nb, 256, 0, st>>>(k, pcm, nullptr, meta, blkflags);
}

void launch_unpack(const void *packed, int bytes_per_sample, int32_t *pcm, unsigned long long n, int bps, int *err, cudaStream_t st)
{
	const unsigned long long threads = (n + 3) / 4;
	const unsigned grid = (unsigned)((threads + 255) / 256);
	if(grid == 0) return;
	if(bytes_per_sample == 2) k_unpack<2><<<grid, 256, 0, st>>>(static_cast<const uint8_t *>(packed), pcm, n, bps, err);
	else k_unpack<3><<<grid, 256, 0, st>>>(static_cast<const uint8_t *>(packed), pcm, n, bps, err);
}

void launch_minbr_flags(const EncK &k, const SubframePlan *plans, const int *blkflags, int nb, int *flags, cudaStream_t st)
{
	k_minbr_flags<<<(nb + 127) / 128, 128, 0, st>>>(k, plans, blkflags, nb, flags);
}

void launch_lpc(const EncK &k, const double *autoc, const DevCand *cands, SigMeta *meta, const uint32_t *sigor, CandDesc *cdesc, int nitems, int autoc_unshifted, cudaStream_t st)
{
	const int total = nitems * k.nwin;
	if(k.max_order <= 8) k_lpc<8><<<(total + 127) / 128, 128, 0, st>>>(k, autoc, cands, meta, sigor, cdesc, nitems, autoc_unshifted);
	else if(k.max_order <= 12) k_lpc<12><<<(total + 127) / 128, 128, 0, st>>>(k, autoc, cands, meta, sigor, cdesc, nitems, autoc_unshifted);
	else k_lpc<32><<<(total + 127) / 128, 128, 0, st>>>(k, autoc, cands, meta, sigor, cdesc, nitems, autoc_unshifted);
}

void launch_search_general(const EncK &k, size_t smem, const int32_t *sig, const SigMeta *meta, const CandDesc *cdesc, SubframePlan *plans, int nitems, cudaStream_t st)
{
	k_search<<<nitems, 128, smem, st>>>(k, sig, meta, cdesc, plans);
}

void launch_emit_general(const EncK &k, size_t smem, const int32_t *sig, const int *blkflags, const SubframePlan *plans, uint8_t *slots, uint32_t *frame_bytes, uint32_t *chan_assign, int nb, cudaStream_t st)
{
	k_emit<<<nb, 256, smem, st>>>(k, sig, blkflags, plans, slots, frame_bytes, chan_assign);
}

void launch_scan(const uint32_t *bytes, int n, unsigned long long *offsets, unsigned long long *running, cudaStream_t st)
{
	k_scan<<<1, 1024, 0, st>>>(bytes, n, offsets, running);
}

void launch_gather(const EncK &k, const uint8_t *slots, const uint32_t *bytes, const unsigned long long *offsets, uint8_t *out, unsigned long long capacity, int *err, int nb, cudaStream_t st)
{
	k_gather<<<nb, 256, 0, st>>>(k, slots, bytes, offsets, out, capacity, err);
}

// fb200_debug_evaluate_lpc: evaluate_candidate (k_search's per-candidate evaluation) on one LPC candidate per CTA; est = its
// estimate, 0xffffffff when the candidate is rejected
__global__ void __launch_bounds__(128) k_debug_evaluate(EncK P, const int32_t *__restrict__ sig, const SigMeta *__restrict__ meta,
                                                        const CandDesc *__restrict__ cands, uint32_t *__restrict__ absr, uint32_t *__restrict__ est)
{
	__shared__ SearchShared S;
	const int c = blockIdx.x;
	if(threadIdx.x == 0) { S.fail = 0; S.best_bits = 0xffffffffu; }
	if(threadIdx.x < FB200_MAX_LPC_ORDER) S.c_qlp[threadIdx.x] = cands[c].qlp[threadIdx.x];
	__syncthreads();
	const CandDesc &D = cands[c];
	evaluate_candidate(P, S, sig + (size_t)c * P.bs, absr + (size_t)c * P.bs, SF_LPC, D.order, D.precision, D.shift, D.wide, D.limit,
	                   meta[c].bps, meta[c].wasted);
	if(threadIdx.x == 0) est[c] = S.best_bits;
}

void launch_debug_evaluate(const EncK &k, const int32_t *sig, const SigMeta *meta, const CandDesc *cands, uint32_t *absr, uint32_t *est, int n)
{
	k_debug_evaluate<<<n, 128>>>(k, sig, meta, cands, absr, est);
}

void launch_debug_log(const double *dx, double *dy, int n) { k_debug_log<<<(n + 255) / 256, 256>>>(dx, dy, n); }

// The dynamic shared-memory opt-in is a per-function, per-device attribute: set it ONCE to the device maximum, so that
// encoders with different blocksizes in one process never lower each other's limit.
void general_kernels_init(int device)
{
	cudaDeviceProp prop;
	cudaGetDeviceProperties(&prop, device);
	cudaFuncSetAttribute(k_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin - 8192);
	cudaFuncSetAttribute(k_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin - 4096);
}

}  // namespace fb200
