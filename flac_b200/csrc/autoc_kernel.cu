// autoc_kernel.cu -- k_autoc3 and its launcher.
#include "autoc_kernel.cuh"

namespace fb200 {

template <int LAGS, int U, int K, int STAGES>
static void autoc3(const EncK &k, const int32_t *sig, const SigMeta *meta, const float *windows, const DevSection *secs, double *autoc, int nitems, cudaStream_t st)
{
	const int groups = (nitems + 31) / 32;
	k_autoc3<LAGS, U, K, STAGES><<<groups * k.nsec, 32, autoc3_smem_bytes<LAGS, U, K, STAGES>(), st>>>(k, sig, meta, windows, secs, autoc, nitems);
}

int autoc_kernel_lags(int lags) { return lags <= 7 ? 7 : lags <= 9 ? 9 : lags <= 13 ? 13 : lags <= 17 ? 17 : 33; }

// warp per 32 chains, asynchronously staged tiles; tile shapes tuned per lag count (DESIGN.md "Kernels")
void launch_autoc3(const EncK &k, const int32_t *sig, const SigMeta *meta, const float *windows, const DevSection *secs, double *autoc, int nitems, cudaStream_t st)
{
	switch(autoc_kernel_lags(k.lags)) {
		case 7: autoc3<7, 28, 2, 4>(k, sig, meta, windows, secs, autoc, nitems, st); break;
		case 9: autoc3<9, 36, 2, 4>(k, sig, meta, windows, secs, autoc, nitems, st); break;
		case 13: autoc3<13, 52, 1, 4>(k, sig, meta, windows, secs, autoc, nitems, st); break;
		case 17: autoc3<17, 68, 1, 3>(k, sig, meta, windows, secs, autoc, nitems, st); break;
		default: autoc3<33, 132, 1, 3>(k, sig, meta, windows, secs, autoc, nitems, st); break;
	}
}

template <int LAGS, int U, int K, int STAGES>
static void autoc4(const EncK &k, const int32_t *pcm, const SigMeta *meta, const float *secwin, int secwin_stride, const DevSection *secs, double *autoc, int nitems, uint32_t *sigor, int or_sec, cudaStream_t st)
{
	const int groups = (nitems + 31) / 32;
	const int mode = k.channels == 1 ? 0 : k.channels == 2 ? 1 : 2;
	const size_t smem = autoc4_smem_bytes<U, K, STAGES>(k.nsig, k.channels, mode);
	if(mode == 0) k_autoc4<LAGS, U, K, STAGES, 0><<<groups * k.nsec, 32, smem, st>>>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec);
	else if(mode == 1) k_autoc4<LAGS, U, K, STAGES, 1><<<groups * k.nsec, 32, smem, st>>>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec);
	else k_autoc4<LAGS, U, K, STAGES, 2><<<groups * k.nsec, 32, smem, st>>>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec);
}

// the same tile shapes as k_autoc3, fed from the caller's interleaved PCM through TMA bulk copies
void launch_autoc4(const EncK &k, const int32_t *pcm, const SigMeta *meta, const float *secwin, int secwin_stride, const DevSection *secs, double *autoc, int nitems, uint32_t *sigor, int or_sec, cudaStream_t st)
{
	switch(autoc_kernel_lags(k.lags)) {
		case 7: autoc4<7, 28, 2, 4>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec, st); break;
		case 9: autoc4<9, 36, 2, 4>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec, st); break;
		case 13: autoc4<13, 52, 1, 4>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec, st); break;
		case 17: autoc4<17, 68, 1, 3>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec, st); break;
		default: autoc4<33, 132, 1, 3>(k, pcm, meta, secwin, secwin_stride, secs, autoc, nitems, sigor, or_sec, st); break;
	}
}

template <int LAGS, int U, int K, int STAGES>
static void autoc4_attrs()
{
	cudaFuncSetAttribute(k_autoc4<LAGS, U, K, STAGES, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
	cudaFuncSetAttribute(k_autoc4<LAGS, U, K, STAGES, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
	cudaFuncSetAttribute(k_autoc4<LAGS, U, K, STAGES, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
}

void autoc4_init(int)
{
	autoc4_attrs<7, 28, 2, 4>(); autoc4_attrs<9, 36, 2, 4>(); autoc4_attrs<13, 52, 1, 4>(); autoc4_attrs<17, 68, 1, 3>(); autoc4_attrs<33, 132, 1, 3>();
}

void autoc3_init(int)
{
	cudaFuncSetAttribute(k_autoc3<33, 132, 1, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)autoc3_smem_bytes<33, 132, 1, 3>());
}

}  // namespace fb200
