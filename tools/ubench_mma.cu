// Micro-benchmark: legacy mma.sync throughput on this GPU - IMMA m16n8k32 (s8), IMMA m16n8k16 (s8),
// HMMA m16n8k16 (f16 -> f32, bf16 -> f32). Each warp keeps NCH independent accumulator chains.
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench_mma tools/ubench_mma.cu
#include <cstdio>
#include <cuda_runtime.h>

template<int OP, int NCH> __global__ void __launch_bounds__(256) k(int *out, int n, unsigned a0, unsigned b0)
{
	unsigned a[4] = { a0 + threadIdx.x, a0 * 3 + 1, a0 ^ 0x55u, a0 + 7 };
	unsigned b[2] = { b0 + threadIdx.x, b0 * 5 + 3 };
	int c[NCH][4];
	float f[NCH][4];
	for(int i = 0; i < NCH; i++) for(int j = 0; j < 4; j++) { c[i][j] = i + j; f[i][j] = 0.0f; }
	for(int it = 0; it < n; it++)
	{
		#pragma unroll
		for(int i = 0; i < NCH; i++)
		{
			if(OP == 0) asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
				: "+r"(c[i][0]), "+r"(c[i][1]), "+r"(c[i][2]), "+r"(c[i][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
			if(OP == 1) asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
				: "+r"(c[i][0]), "+r"(c[i][1]), "+r"(c[i][2]), "+r"(c[i][3]) : "r"(a[0]), "r"(a[1]), "r"(b[0]));
			if(OP == 2) asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
				: "+f"(f[i][0]), "+f"(f[i][1]), "+f"(f[i][2]), "+f"(f[i][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
			if(OP == 3) asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
				: "+f"(f[i][0]), "+f"(f[i][1]), "+f"(f[i][2]), "+f"(f[i][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
			if(OP == 4) asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
				: "+f"(f[i][0]), "+f"(f[i][1]), "+f"(f[i][2]), "+f"(f[i][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
		}
	}
	int s = 0; float t = 0;
	for(int i = 0; i < NCH; i++) for(int j = 0; j < 4; j++) { s += c[i][j]; t += f[i][j]; }
	out[blockIdx.x * blockDim.x + threadIdx.x] = s + (int) t;
}

template<int OP, int NCH> void run(const char *name, double macs_per_mma, int ctas_per_sm)
{
	int *d; cudaMalloc(&d, 148 * 8 * 256 * 4);
	cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
	const int n = 4000;
	k<OP, NCH><<<148 * ctas_per_sm, 256>>>(d, 100, 0, 0);
	cudaEventRecord(e0);
	k<OP, NCH><<<148 * ctas_per_sm, 256>>>(d, n, 0, 0);
	cudaEventRecord(e1); cudaEventSynchronize(e1);
	float ms; cudaEventElapsedTime(&ms, e0, e1);
	const double mmas = (double) 148 * ctas_per_sm * 8 * n * NCH;
	printf("%-26s chains %d, %d warps/SM: %8.1f TMAC/s  %7.1f MAC/clk/SM  %6.2f clk per mma per SM sub-partition (1.965 GHz)\n",
		name, NCH, 8 * ctas_per_sm, mmas * macs_per_mma / ms / 1e9, mmas * macs_per_mma / ms / 1e6 / 148 / 1.965,
		ms * 1e-3 * 1.965e9 / (mmas / 148 / 4));
	cudaFree(d);
}

int main()
{
	run<0, 8>("IMMA m16n8k32 s8", 4096, 4);
	run<0, 2>("IMMA m16n8k32 s8", 4096, 4);
	run<0, 8>("IMMA m16n8k32 s8", 4096, 1);
	run<1, 8>("IMMA m16n8k16 s8", 2048, 4);
	run<2, 8>("HMMA m16n8k16 f16->f32", 2048, 4);
	run<2, 2>("HMMA m16n8k16 f16->f32", 2048, 4);
	run<3, 8>("HMMA m16n8k16 bf16->f32", 2048, 4);
	run<4, 8>("QMMA m16n8k32 e4m3->f32", 4096, 4);
	return 0;
}
