// Micro-benchmark (development aid): cost of random sector gathers through the LSU on H100.
//   A: one lane reads one 32 B record with two LDG.128 back to back (the mask loads of csrc/; sm_90 has no LDG.256)
//   B: two adjacent lanes read the halves of one 32 B record  (16 records / warp instruction, LDG.128)
//   C: one lane reads one 16 B record with LDG.128
//   D: one lane reads one  8 B record with LDG.64
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/mb tools/microbench_gather.cu && /tmp/mb
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
typedef unsigned long long u64;
__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

template <int MODE>
__global__ void __launch_bounds__(256) k(const u64 *__restrict__ tab, const uint32_t *__restrict__ idx, int64_t n, uint32_t mask, u64 *out) {
	u64 acc = 0;
	int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	int64_t stride = (int64_t)gridDim.x * blockDim.x;
	if (MODE == 1) { // pairs of lanes share a record: thread t handles record t/2, half t&1
		for (int64_t i = tid; i < 2 * n; i += stride) {
			uint32_t r = idx[i >> 1] & mask;
			const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(tab + (int64_t)r * 4 + 2 * (i & 1)));
			acc |= v.x ^ v.y;
		}
	} else {
		for (int64_t i = tid; i < n; i += stride) {
			uint32_t r = idx[i] & mask;
			if (MODE == 0) {
				u64 a, b, c, d;
				asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%4];\n\tld.global.nc.v2.u64 {%2,%3}, [%4+16];"
				             : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(tab + (int64_t)r * 4));
				acc |= a ^ b ^ c ^ d;
			} else if (MODE == 2) {
				const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(tab + (int64_t)r * 2));
				acc |= v.x ^ v.y;
			} else {
				acc |= __ldg(tab + r);
			}
		}
	}
	if (acc == 0x1234567) out[0] = acc;
}
__global__ void fill(uint32_t *idx, int64_t n) { for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) idx[i] = mix((uint32_t)i); }

int main() {
	const int64_t n = 64 << 20;
	uint32_t *idx; u64 *tab, *out;
	cudaMalloc(&idx, n * 4); cudaMalloc(&out, 8);
	fill<<<1184, 256>>>(idx, n);
	for (int mb : {16, 64, 256}) {
		size_t bytes = (size_t)mb << 20;
		cudaMalloc(&tab, bytes); cudaMemset(tab, 1, bytes);
		cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
		const char *names[4] = {"A 2 x LDG.128 32B/lane", "B 2 lanes x LDG.128 (32B rec)", "C LDG.128 16B/lane", "D LDG.64 8B/lane"};
		for (int mode = 0; mode < 4; mode++) {
			uint32_t recbytes = mode <= 1 ? 32 : (mode == 2 ? 16 : 8);
			uint32_t mask = (uint32_t)(bytes / recbytes) - 1;
			float best = 1e9;
			for (int rep = 0; rep < 5; rep++) {
				cudaEventRecord(a);
				if (mode == 0) k<0><<<132 * 8, 256>>>(tab, idx, n, mask, out);
				if (mode == 1) k<1><<<132 * 8, 256>>>(tab, idx, n, mask, out);
				if (mode == 2) k<2><<<132 * 8, 256>>>(tab, idx, n, mask, out);
				if (mode == 3) k<3><<<132 * 8, 256>>>(tab, idx, n, mask, out);
				cudaEventRecord(b); cudaEventSynchronize(b);
				float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
			}
			printf("table %3d MB  %-32s %7.3f ms  %6.1f G records/s\n", mb, names[mode], best, n / best / 1e6);
		}
		cudaFree(tab);
	}
	return 0;
}
