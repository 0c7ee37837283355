// Micro-benchmark: issue throughput of IMAD, IDP.2A (dp2a), IADD3, FFMA on this GPU.
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o /tmp/ubench tools/ubench_pipes.cu
#include <cstdio>
#include <cuda_runtime.h>
template<int OP> __global__ void k(int *out, int n, int a0, int b0)
{
	int a[8], b = b0 + threadIdx.x;
	float f[8], g = (float) b0;
	for(int i = 0; i < 8; i++) { a[i] = a0 + i + threadIdx.x; f[i] = (float) a[i]; }
	for(int it = 0; it < n; it++)
	{
		#pragma unroll
		for(int i = 0; i < 8; i++)
		{
			if(OP == 0) a[i] = a[i] * b + a[(i + 1) & 7];
			if(OP == 1) a[i] = __dp2a_lo(a[(i + 1) & 7], b, a[i]);
			if(OP == 2) a[i] = a[i] + b + a[(i + 1) & 7];
			if(OP == 3) f[i] = f[i] * g + f[(i + 1) & 7];
			if(OP == 4) a[i] = __dp4a(a[(i + 1) & 7], b, a[i]);
		}
	}
	int s = 0; float t = 0;
	for(int i = 0; i < 8; i++) { s += a[i]; t += f[i]; }
	out[blockIdx.x * blockDim.x + threadIdx.x] = s + (int) t;
}
template<int OP> void run(const char *name)
{
	int *d; cudaMalloc(&d, 148 * 8 * 256 * 4);
	cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
	const int n = 20000;
	k<OP><<<148 * 8, 256>>>(d, 100, 1, 3);
	cudaEventRecord(e0);
	k<OP><<<148 * 8, 256>>>(d, n, 1, 3);
	cudaEventRecord(e1); cudaEventSynchronize(e1);
	float ms; cudaEventElapsedTime(&ms, e0, e1);
	double ops = (double) 148 * 8 * 256 * n * 8;
	printf("%-8s %.1f Gops/s  (%.1f lane-ops/clk/SM at 1.965 GHz)\n", name, ops / ms / 1e6, ops / ms / 1e6 / 148 / 1.965);
	cudaFree(d);
}
int main() { run<0>("IMAD"); run<1>("DP2A"); run<2>("IADD3"); run<3>("FFMA"); run<4>("DP4A"); return 0; }
