// Micro-benchmark: FP64 / conversion pipe rates and latencies on this GPU (inputs to k_autoc's roofline).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o fp64_rates fp64_rates.cu && ./fp64_rates
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int OP, int CHAINS>
__global__ void k_tput(double *out, const float *in, int iters)
{
	double acc[CHAINS];
	float f[CHAINS];
	int iv[CHAINS];
	const double a = (double)in[threadIdx.x & 7] , b = (double)in[8 + (threadIdx.x & 7)];
#pragma unroll
	for(int c = 0; c < CHAINS; c++) { acc[c] = (double)in[c] + threadIdx.x; f[c] = in[c] + threadIdx.x; iv[c] = (int)in[c] + threadIdx.x; }
	for(int i = 0; i < iters; i++) {
#pragma unroll
		for(int c = 0; c < CHAINS; c++) {
			if(OP == 0) acc[c] = fma(acc[c], a, b);                 // DFMA
			else if(OP == 1) acc[c] = __dadd_rn(acc[c], a);         // DADD
			else if(OP == 2) acc[c] = __dmul_rn(acc[c], a);         // DMUL
			else if(OP == 3) { f[c] = (float)((double)f[c] + b); }  // F2D + DADD + D2F
			else if(OP == 4) { acc[c] += (double)f[c]; f[c] = __int_as_float(__float_as_int(f[c]) + 1); }  // F2F.F64.F32 + DADD + IADD
			else if(OP == 5) { f[c] += (float)iv[c]; iv[c] += 3; }  // I2F + FADD + IADD
			else if(OP == 6) f[c] = fmaf(f[c], (float)a, (float)b); // FFMA
		}
	}
	double s = 0;
#pragma unroll
	for(int c = 0; c < CHAINS; c++) s += acc[c] + f[c] + iv[c];
	out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int OP, int CHAINS>
static void run(const char *name, int ops_per_iter_chain, int blocks, int threads, double *d_out, float *d_in, int sms, double mhz)
{
	const int iters = 4096;
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0); cudaEventCreate(&e1);
	k_tput<OP, CHAINS><<<blocks, threads>>>(d_out, d_in, iters);
	cudaEventRecord(e0);
	k_tput<OP, CHAINS><<<blocks, threads>>>(d_out, d_in, iters);
	cudaEventRecord(e1);
	cudaEventSynchronize(e1);
	float ms = 0;
	cudaEventElapsedTime(&ms, e0, e1);
	const double ops = (double)blocks * threads * iters * CHAINS * ops_per_iter_chain;
	printf("%-34s chains=%d grid=%dx%d  %.3f ms  %.2f Tops/s  %.1f thread-ops/clk/SM (at %.0f MHz)\n", name, CHAINS, blocks, threads, ms, ops / ms * 1e-9,
	       ops / (ms * 1e-3) / (mhz * 1e6) / sms, mhz);
}

int main()
{
	cudaDeviceProp p;
	cudaGetDeviceProperties(&p, 0);
	int khz = 0;
	cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
	const double mhz = khz / 1000.0;
	printf("%s  SMs=%d  clock=%.0f MHz\n", p.name, p.multiProcessorCount, mhz);
	double *d_out; float *d_in;
	cudaMalloc(&d_out, sizeof(double) * p.multiProcessorCount * 8 * 1024 * 2);
	float h[16]; for(int i = 0; i < 16; i++) h[i] = 1.0f + i * 1e-3f;
	cudaMalloc(&d_in, sizeof h); cudaMemcpy(d_in, h, sizeof h, cudaMemcpyHostToDevice);
	const int sms = p.multiProcessorCount;
	// throughput: full occupancy
	run<0, 8>("DFMA throughput", 1, sms * 8, 256, d_out, d_in, sms, mhz);
	run<1, 8>("DADD throughput", 1, sms * 8, 256, d_out, d_in, sms, mhz);
	run<2, 8>("DMUL throughput", 1, sms * 8, 256, d_out, d_in, sms, mhz);
	run<3, 8>("F2D+DADD+D2F (3 ops)", 3, sms * 8, 256, d_out, d_in, sms, mhz);
	run<4, 8>("F2D+DADD (+IADD) (2 ops)", 2, sms * 8, 256, d_out, d_in, sms, mhz);
	run<5, 8>("I2F+FADD (+IADD) (2 ops)", 2, sms * 8, 256, d_out, d_in, sms, mhz);
	run<6, 8>("FFMA throughput", 1, sms * 8, 256, d_out, d_in, sms, mhz);
	// latency: one warp per SM, one chain  -> cycles per dependent op = 1 / (ops/clk/SM / 32)
	run<0, 1>("DFMA dependent, 1 warp/SM", 1, sms, 32, d_out, d_in, sms, mhz);
	run<1, 1>("DADD dependent, 1 warp/SM", 1, sms, 32, d_out, d_in, sms, mhz);
	run<6, 1>("FFMA dependent, 1 warp/SM", 1, sms, 32, d_out, d_in, sms, mhz);
	// one warp per SMSP, 9 and 13 independent chains (k_autoc's situation at -5 / -8)
	run<0, 9>("DFMA 9 chains, 4 warps/SM", 1, sms, 128, d_out, d_in, sms, mhz);
	run<0, 13>("DFMA 13 chains, 4 warps/SM", 1, sms, 128, d_out, d_in, sms, mhz);
	run<0, 9>("DFMA 9 chains, 8 warps/SM", 1, sms * 2, 128, d_out, d_in, sms, mhz);
	run<0, 9>("DFMA 9 chains, 16 warps/SM", 1, sms * 4, 128, d_out, d_in, sms, mhz);
	cudaDeviceSynchronize();
	printf("last error: %s\n", cudaGetErrorString(cudaGetLastError()));
	return 0;
}
