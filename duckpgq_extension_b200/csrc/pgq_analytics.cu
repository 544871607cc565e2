// pgq_analytics.cu -- the reference's other consumers of the CSR on the device, bit for bit:
//   local_clustering_coefficient  local_clustering_coefficient.cpp:41-70
//   pagerank                      pagerank.cpp:31-84
//   weakly_connected_component    weakly_connected_component.cpp:37-104
// sm_90a only.  In all three the reference's v_size is CSR::vsize = n + 2 (csr_creation.cpp:30): the two entries
// behind the vertices have no edges and take part where the reference lets them.  DESIGN.md section 3 gives the
// arguments for exactness; in short:
//   - LCC only tests set membership, so it runs on the internal ids.
//   - PageRank's sums are left folds in the reference's order: temp[t] over t's in-edges by ascending ORIGINAL
//     source id (an in-CSC in that order is built for the computation), the dangling total over the out-degree-0
//     entries by ascending original id (one warp, sequentially).  No FMA contraction anywhere.
//   - WCC's labels depend only on the ordered sequence of merge edges, which is the minimum spanning forest under
//     "weight = reference CSR position": Boruvka finds it on the device, the host replays Link over it in order.
// PageRank and WCC are computed once per CSR, on the first call, and answered from a host copy afterwards.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <vector>

#include "pgq_internal.h"

#define AN_FULL 0xffffffffu
// Workspace slots: 28-30 hold the BFS lane-mask arrays, whose zero rows a workspace remembers between calls
// (pgq_bfs.cu, clean_from), and 14-15 the radix sort's scratch; this file uses the other slots as scratch only.
#define LCC_SMEM 4096 // out-lists up to this length are sorted in shared memory; longer ones use a bitmap over n

static inline unsigned an_grid(int64_t count, int threads, int64_t cap) {
	const int64_t g = (count + threads - 1) / threads;
	return (unsigned)std::max<int64_t>(1, std::min<int64_t>(g, cap));
}

// ---- shared: the reference's CSR offsets ------------------------------------------------------------------------
// odeg[v] = out-degree of ORIGINAL id v for v < n, 0 for the two entries n, n+1 and for the scan's total slot
__global__ void k_an_odeg(const int32_t *__restrict__ off, const int32_t *__restrict__ perm, int64_t n, int32_t *odeg) {
	for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n + 3; v += (int64_t)gridDim.x * blockDim.x) {
		odeg[v] = (v < n) ? off[perm[v] + 1] - off[perm[v]] : 0;
	}
}

// ref_off[v] = v[v] of the reference's layout, v in [0, n + 2]; ref_off[n + 2] = m
static int ref_offsets(pgq_csr *csr, Workspace *ws, cudaStream_t s, int32_t **ref_off, int64_t *launches) {
	const int64_t n = csr->n;
	int32_t *ro, *scan_tmp;
	PGQ_TRY(pgq_ws_reserve(ws, WS_AN_REF_OFF, (size_t)(n + 3) * sizeof(int32_t), (void **)&ro));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AN_SCAN, pgq_scan_tmp_elems(n + 3) * sizeof(int32_t), (void **)&scan_tmp));
	k_an_odeg<<<an_grid(n + 3, 256, (int64_t)csr->ctx->sm_count * 8), 256, 0, s>>>(csr->out.off, csr->perm, n, ro);
	PGQ_CUDA(cudaGetLastError());
	PGQ_TRY(pgq_scan_exclusive_i32(ro, ro, n + 3, scan_tmp, s));
	*launches += 2;
	*ref_off = ro;
	return PGQ_OK;
}

static int bits_for(int64_t count) {
	int b = 1;
	while (b < 31 && ((int64_t)1 << b) < count) {
		b++;
	}
	return b;
}

// In reference order: folds values[ids[b]], values[ids[b+1]], ... values[ids[e-1]] into 0.0, one dependent add
// per element.  The lanes stage the next 32 values while the current 32 are folded, and a full group of 32 is
// gathered from the lanes before its adds, so that the chain is bound by the adds alone; every lane ends with the sum.
__device__ __forceinline__ double warp_fold(const int32_t *__restrict__ ids, int64_t b, int64_t e,
                                            const double *__restrict__ values, int lane) {
	double acc = 0.0;
	double x = (b + lane < e) ? values[ids[b + lane]] : 0.0;
	for (int64_t c = b; c < e; c += 32) {
		const int64_t nx = c + 32 + lane;
		const double y = (nx < e) ? values[ids[nx]] : 0.0;
		if (e - c >= 32) {
			double g[32];
#pragma unroll
			for (int j = 0; j < 32; j++) {
				g[j] = __shfl_sync(AN_FULL, x, j);
			}
#pragma unroll
			for (int j = 0; j < 32; j++) {
				acc = __dadd_rn(acc, g[j]);
			}
		} else {
			for (int j = 0; j < (int)(e - c); j++) {
				acc = __dadd_rn(acc, __shfl_sync(AN_FULL, x, j));
			}
		}
		x = y;
	}
	return acc;
}

// =================================================================================================================
// local_clustering_coefficient
// =================================================================================================================
__device__ __forceinline__ bool sorted_contains(const int32_t *list, int k, int32_t x) {
	int lo = 0, hi = k;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (list[mid] < x) {
			lo = mid + 1;
		} else {
			hi = mid;
		}
	}
	return lo < k && list[lo] == x;
}

__device__ __forceinline__ u64 block_sum_u64(u64 x, u64 *red) {
	for (int d = 16; d > 0; d >>= 1) {
		x += __shfl_xor_sync(AN_FULL, x, d);
	}
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	__syncthreads();
	if (lane == 0) {
		red[warp] = x;
	}
	__syncthreads();
	u64 t = 0;
	if (threadIdx.x == 0) {
		for (int w = 0; w < (int)(blockDim.x >> 5); w++) {
			t += red[w];
		}
	}
	return t; // valid in thread 0
}

// (float)count / (k * (k - 1.0f)) in float, as local_clustering_coefficient.cpp:64-65
__device__ __forceinline__ float lcc_value(u64 count, int k) {
	const float kf = (float)k;
	return __fdiv_rn(__ll2float_rn((long long)count), __fmul_rn(kf, __fsub_rn(kf, 1.0f)));
}

// One block per row.  Out-lists of at most LCC_SMEM entries are sorted in shared memory and every entry of every
// neighbour's list is looked up there; longer ones are queued for the bitmap path (big_rows).
__global__ void __launch_bounds__(256) k_lcc_rows(int64_t p, const int64_t *__restrict__ src,
                                                  const uint8_t *__restrict__ src_valid, const int32_t *__restrict__ perm,
                                                  const int32_t *__restrict__ off, const int32_t *__restrict__ adj,
                                                  float *out, uint8_t *out_valid, int32_t *big_rows, int *big_count) {
	__shared__ int32_t list[LCC_SMEM];
	__shared__ u64 red[8];
	for (int64_t row = blockIdx.x; row < p; row += gridDim.x) {
		if (src_valid && !src_valid[row]) {
			if (threadIdx.x == 0) {
				out[row] = 0.0f;
				out_valid[row] = 0;
			}
			continue;
		}
		const int ps = perm[src[row]];
		const int b = off[ps], k = off[ps + 1] - b;
		if (k < 2 || k > LCC_SMEM) {
			if (threadIdx.x == 0) {
				out[row] = 0.0f;
				out_valid[row] = 1;
				if (k >= 2) {
					big_rows[atomicAdd(big_count, 1)] = (int32_t)row;
				}
			}
			continue;
		}
		int size = 32;
		while (size < k) {
			size <<= 1;
		}
		__syncthreads(); // (the previous row's lookups are done)
		for (int i = threadIdx.x; i < size; i += blockDim.x) {
			list[i] = (i < k) ? adj[b + i] : 0x7fffffff;
		}
		__syncthreads();
		for (int w = 2; w <= size; w <<= 1) { // bitonic sort, ascending
			for (int j = w >> 1; j > 0; j >>= 1) {
				for (int i = threadIdx.x; i < size; i += blockDim.x) {
					const int q = i ^ j;
					if (q > i) {
						const int32_t a = list[i], c = list[q];
						if (((i & w) == 0) == (a > c)) {
							list[i] = c;
							list[q] = a;
						}
					}
				}
				__syncthreads();
			}
		}
		const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
		u64 count = 0;
		for (int i = warp; i < k; i += nwarps) { // every neighbour, with multiplicity
			const int u = list[i];
			for (int j = off[u] + lane; j < off[u + 1]; j += 32) {
				count += sorted_contains(list, k, adj[j]);
			}
		}
		const u64 total = block_sum_u64(count, red);
		if (threadIdx.x == 0) {
			out[row] = lcc_value(total, k);
			out_valid[row] = 1;
		}
	}
}

// Bitmap path of the long rows, a group at a time: row i0 + blockIdx.y uses bitmap blockIdx.y (`words` words each).
// Mark the row's neighbours (set) or clear the words it marked (!set) ...
__global__ void k_lcc_big_mark(int i0, const int32_t *__restrict__ big_rows, const int64_t *__restrict__ src,
                               const int32_t *__restrict__ perm, const int32_t *__restrict__ off,
                               const int32_t *__restrict__ adj, uint32_t *bitmaps, int64_t words, bool set) {
	const int ps = perm[src[big_rows[i0 + blockIdx.y]]];
	const int b = off[ps], k = off[ps + 1] - b;
	uint32_t *bitmap = bitmaps + (int64_t)blockIdx.y * words;
	for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < k; j += (int64_t)gridDim.x * blockDim.x) {
		const int32_t u = adj[b + j];
		if (set) {
			atomicOr(&bitmap[u >> 5], 1u << (u & 31));
		} else {
			bitmap[u >> 5] = 0;
		}
	}
}

// ... and count, a warp per neighbour entry
__global__ void __launch_bounds__(256) k_lcc_big_count(int i0, const int32_t *__restrict__ big_rows,
                                                       const int64_t *__restrict__ src, const int32_t *__restrict__ perm,
                                                       const int32_t *__restrict__ off, const int32_t *__restrict__ adj,
                                                       const uint32_t *__restrict__ bitmaps, int64_t words, u64 *big_cnt) {
	__shared__ u64 red[8];
	const int i = i0 + blockIdx.y;
	const uint32_t *bitmap = bitmaps + (int64_t)blockIdx.y * words;
	const int ps = perm[src[big_rows[i]]];
	const int b = off[ps], k = off[ps + 1] - b;
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	u64 count = 0;
	for (int64_t t = warp; t < k; t += nwarps) {
		const int u = adj[b + t];
		for (int j = off[u] + lane; j < off[u + 1]; j += 32) {
			const int32_t w = adj[j];
			count += (bitmap[w >> 5] >> (w & 31)) & 1u;
		}
	}
	const u64 total = block_sum_u64(count, red);
	if (threadIdx.x == 0 && total) {
		atomicAdd(&big_cnt[i], total);
	}
}

__global__ void k_lcc_big_finish(int nbig, const int32_t *__restrict__ big_rows, const int64_t *__restrict__ src,
                                 const int32_t *__restrict__ perm, const int32_t *__restrict__ off,
                                 const u64 *__restrict__ big_cnt, float *out) {
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nbig; i += gridDim.x * blockDim.x) {
		const int64_t row = big_rows[i];
		const int ps = perm[src[row]];
		out[row] = lcc_value(big_cnt[i], off[ps + 1] - off[ps]);
	}
}

extern "C" int pgq_local_clustering_coefficient(pgq_csr *csr, int64_t p, const int64_t *src, const uint8_t *src_valid,
                                                float *out, uint8_t *out_valid, pgq_stats *stats) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (p < 0 || (p > 0 && (!src || !out || !out_valid))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (p >= 0x7fffffffLL) {
		return pgq_fail(PGQ_ERR_RANGE, "too many rows in one call");
	}
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	// the reference reads v[src] and v[src + 1] unchecked (local_clustering_coefficient.cpp:50): an id outside
	// [0, n) is refused here (DESIGN.md section 7)
	for (int64_t r = 0; r < p; r++) {
		if ((!src_valid || src_valid[r]) && (src[r] < 0 || src[r] >= csr->n)) {
			return pgq_fail(PGQ_ERR_RANGE, "local_clustering_coefficient: vertex id %lld outside [0,%lld)",
			                (long long)src[r], (long long)csr->n);
		}
	}
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	if (p == 0) {
		if (stats) {
			*stats = st;
		}
		return PGQ_OK;
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	int64_t *d_src;
	uint8_t *d_sv, *d_ov;
	float *d_out;
	int32_t *big_rows;
	int *big_count, *h_big;
	u64 *big_cnt;
	uint32_t *bitmap;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	PGQ_TRY(pgq_ws_reserve(ws, WS_LCC_OUT, (size_t)p * sizeof(float), (void **)&d_out));
	PGQ_TRY(pgq_ws_reserve(ws, WS_LCC_OUT_VALID, (size_t)p, (void **)&d_ov));
	PGQ_TRY(pgq_ws_reserve(ws, WS_LCC_BIG_ROWS, (size_t)p * sizeof(int32_t) + 64, (void **)&big_rows));
	PGQ_TRY(pgq_ws_reserve(ws, WS_LCC_BIG_CNT, (size_t)p * sizeof(u64), (void **)&big_cnt));
	PGQ_TRY(pgq_ws_pinned(ws, 256, (void **)&h_big));
	big_count = big_rows + p;
	cudaEventRecord(ws->ev_begin, s);
	PGQ_TRY(stage_column(ws, WS_LCC_SRC, src, b8, (const void **)&d_src));
	PGQ_TRY(stage_column(ws, WS_LCC_SRC_VALID, src_valid, (size_t)p, (const void **)&d_sv));
	st.h2d_bytes = (int64_t)b8 + (src_valid ? p : 0);
	cudaMemsetAsync(big_count, 0, sizeof(int), s);
	k_lcc_rows<<<(unsigned)std::min<int64_t>(p, (int64_t)csr->ctx->sm_count * 16), 256, 0, s>>>(
	    p, d_src, d_sv, csr->perm, csr->out.off, csr->out.adj, d_out, d_ov, big_rows, big_count);
	st.kernel_launches++;
	cudaError_t e = cudaMemcpyAsync(h_big, big_count, sizeof(int), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) {
		e = cudaStreamSynchronize(s);
	}
	if (e != cudaSuccess) {
		return pgq_fail(PGQ_ERR_CUDA, "local_clustering_coefficient failed: %s", cudaGetErrorString(e));
	}
	const int nbig = *h_big;
	if (nbig > 0) {
		// one bitmap per row of a group, as many rows as 256 MB of bitmaps hold (at most 65535, the grid's y limit);
		// zeroed once, and after a group only the words it marked are cleared again
		const int64_t words = csr->n / 32 + 1;
		const int group = (int)std::max<int64_t>(
		    1, std::min<int64_t>({(int64_t)nbig, ((int64_t)256 << 20) / (words * 4), (int64_t)65535}));
		PGQ_TRY(pgq_ws_reserve(ws, WS_LCC_BITMAP, (size_t)(group * words) * sizeof(uint32_t), (void **)&bitmap));
		cudaMemsetAsync(bitmap, 0, (size_t)(group * words) * sizeof(uint32_t), s);
		cudaMemsetAsync(big_cnt, 0, (size_t)nbig * sizeof(u64), s);
		const unsigned gx_mark = (unsigned)std::max(1, csr->ctx->sm_count * 4 / group);
		const unsigned gx_count = (unsigned)std::max(4, csr->ctx->sm_count * 8 / group);
		for (int i0 = 0; i0 < nbig; i0 += group) {
			const unsigned gy = (unsigned)std::min(group, nbig - i0);
			k_lcc_big_mark<<<dim3(gx_mark, gy), 256, 0, s>>>(i0, big_rows, d_src, csr->perm, csr->out.off, csr->out.adj,
			                                                 bitmap, words, true);
			k_lcc_big_count<<<dim3(gx_count, gy), 256, 0, s>>>(i0, big_rows, d_src, csr->perm, csr->out.off,
			                                                   csr->out.adj, bitmap, words, big_cnt);
			k_lcc_big_mark<<<dim3(gx_mark, gy), 256, 0, s>>>(i0, big_rows, d_src, csr->perm, csr->out.off, csr->out.adj,
			                                                 bitmap, words, false);
			st.kernel_launches += 3;
		}
		k_lcc_big_finish<<<an_grid(nbig, 128, 1024), 128, 0, s>>>(nbig, big_rows, d_src, csr->perm, csr->out.off, big_cnt,
		                                                          d_out);
		st.kernel_launches++;
	}
	cudaMemcpyAsync(out, d_out, (size_t)p * sizeof(float), cudaMemcpyDeviceToHost, s);
	cudaMemcpyAsync(out_valid, d_ov, (size_t)p, cudaMemcpyDeviceToHost, s);
	cudaEventRecord(ws->ev_end, s);
	st.d2h_bytes = (int64_t)p * (int64_t)(sizeof(float) + 1);
	e = cudaStreamSynchronize(s);
	if (e != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) {
		return pgq_fail(PGQ_ERR_CUDA, "local_clustering_coefficient failed: %s", cudaGetErrorString(e));
	}
	g.settled = true;
	float ms = 0.0f;
	cudaEventElapsedTime(&ms, ws->ev_begin, ws->ev_end);
	st.total_ms = ms;
	cudaGetLastError();
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

// =================================================================================================================
// pagerank
// =================================================================================================================
// the out-edges in the reference's CSR order as (key = target, value = source), original ids: row r's j-th edge goes
// to reference position ref_off[inv[r]] + j
__global__ void k_pr_ref_edges(const int32_t *__restrict__ off, const int32_t *__restrict__ adj,
                               const int32_t *__restrict__ inv, int64_t n, const int32_t *__restrict__ ref_off,
                               int32_t *__restrict__ key, int32_t *__restrict__ val) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t r = warp; r < n; r += nwarps) {
		const int32_t a = inv[r];
		const int b = off[r], len = off[r + 1] - b, base = ref_off[a];
		for (int j = lane; j < len; j += 32) {
			key[base + j] = inv[adj[b + j]];
			val[base + j] = a;
		}
	}
}

__global__ void k_pr_histogram(const int32_t *__restrict__ keys, int64_t count, int32_t *hist) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
		atomicAdd(&hist[keys[i]], 1);
	}
}

// rank = 1 / vsize (pagerank.cpp:31), contrib = rank / out-degree; flag = 1 for the dangling entries
__global__ void k_pr_init(int64_t vsize, const int32_t *__restrict__ ref_off, double *rank, double *contrib,
                          int32_t *dangling_flag) {
	const double r0 = __ddiv_rn(1.0, (double)vsize);
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= vsize; i += (int64_t)gridDim.x * blockDim.x) {
		if (i == vsize) {
			dangling_flag[i] = 0;
			continue;
		}
		const int deg = ref_off[i + 1] - ref_off[i];
		rank[i] = r0;
		contrib[i] = deg > 0 ? __ddiv_rn(r0, (double)deg) : 0.0;
		dangling_flag[i] = deg == 0;
	}
}

// dangling[pos[i]] = rank[i] for the out-degree-0 entries: their ranks, contiguous, in ascending original id
__global__ void k_pr_dangling_stage(int64_t vsize, const int32_t *__restrict__ ref_off, const int32_t *__restrict__ pos,
                                    const double *__restrict__ rank, double *dangling) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vsize; i += (int64_t)gridDim.x * blockDim.x) {
		if (ref_off[i + 1] == ref_off[i]) {
			dangling[pos[i]] = rank[i];
		}
	}
}

// total_dangling_rank (pagerank.cpp:49-61): one warp folds the staged dangling ranks in order (ascending original
// id, n and n + 1 last).  The values are contiguous, and the lanes hold the next 128 of them while the current 128
// are added, so the chain is bound by the dependent adds rather than by the loads.
#define PR_FOLD_GROUPS 4
__global__ void k_pr_dangling_fold(const double *__restrict__ dangling, int64_t count, double *total) {
	const int lane = threadIdx.x & 31;
	double acc = 0.0, cur[PR_FOLD_GROUPS];
#pragma unroll
	for (int q = 0; q < PR_FOLD_GROUPS; q++) {
		const int64_t i = q * 32 + lane;
		cur[q] = i < count ? dangling[i] : 0.0;
	}
	for (int64_t c = 0; c < count; c += 32 * PR_FOLD_GROUPS) {
		double nxt[PR_FOLD_GROUPS];
#pragma unroll
		for (int q = 0; q < PR_FOLD_GROUPS; q++) {
			const int64_t i = c + 32 * PR_FOLD_GROUPS + q * 32 + lane;
			nxt[q] = i < count ? dangling[i] : 0.0;
		}
#pragma unroll
		for (int q = 0; q < PR_FOLD_GROUPS; q++) {
			const int64_t g0 = c + q * 32;
			if (count - g0 >= 32) {
				double g[32];
#pragma unroll
				for (int j = 0; j < 32; j++) {
					g[j] = __shfl_sync(AN_FULL, cur[q], j);
				}
#pragma unroll
				for (int j = 0; j < 32; j++) {
					acc = __dadd_rn(acc, g[j]);
				}
			} else {
				for (int j = 0; j < (int)max((int64_t)0, count - g0); j++) {
					acc = __dadd_rn(acc, __shfl_sync(AN_FULL, cur[q], j));
				}
			}
		}
#pragma unroll
		for (int q = 0; q < PR_FOLD_GROUPS; q++) {
			cur[q] = nxt[q];
		}
	}
	if (lane == 0) {
		*total = acc;
	}
}

// temp[t] = left fold of contrib[s] over t's in-edges by ascending original source (a warp per target)
__global__ void __launch_bounds__(256) k_pr_pull(int64_t vsize, const int32_t *__restrict__ in_off,
                                                 const int32_t *__restrict__ in_src, const double *__restrict__ contrib,
                                                 double *temp) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t t = warp; t < vsize; t += nwarps) {
		const double acc = warp_fold(in_src, in_off[t], in_off[t + 1], contrib, lane);
		if (lane == 0) {
			temp[t] = acc;
		}
	}
}

// temp[i] = (1 - d) / vsize + d * (temp[i] + correction), max_delta = max |temp[i] - rank[i]| (pagerank.cpp:64-69),
// without contraction; also the next iteration's contributions and staged dangling ranks.  The deltas are >= 0, so their bit patterns order
// like their values and the max-reduction is exact.
__global__ void __launch_bounds__(256) k_pr_update(int64_t vsize, const int32_t *__restrict__ ref_off,
                                                   const double *__restrict__ rank, double *temp, double *contrib,
                                                   const int32_t *__restrict__ dangling_pos, double *dangling,
                                                   const double *__restrict__ total_dangling, u64 *max_bits) {
	const double vs = (double)vsize;
	const double base = __ddiv_rn(__dsub_rn(1.0, 0.85), vs);
	const double corr = __ddiv_rn(*total_dangling, vs);
	u64 mx = 0;
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vsize; i += (int64_t)gridDim.x * blockDim.x) {
		const double nr = __dadd_rn(base, __dmul_rn(0.85, __dadd_rn(temp[i], corr)));
		const u64 d = (u64)__double_as_longlong(fabs(__dsub_rn(nr, rank[i])));
		mx = d > mx ? d : mx;
		temp[i] = nr;
		const int deg = ref_off[i + 1] - ref_off[i];
		contrib[i] = deg > 0 ? __ddiv_rn(nr, (double)deg) : 0.0;
		if (deg == 0) {
			dangling[dangling_pos[i]] = nr;
		}
	}
	for (int d = 16; d > 0; d >>= 1) {
		const u64 o = __shfl_xor_sync(AN_FULL, mx, d);
		mx = o > mx ? o : mx;
	}
	if ((threadIdx.x & 31) == 0 && mx) {
		atomicMax(max_bits, mx);
	}
}

// Runs PageRank to convergence and keeps the ranks of all vsize entries in csr->pr_rank (called under csr->mu).
static int pagerank_compute(pgq_csr *csr, Workspace *ws, pgq_stats *st) {
	cudaStream_t s = ws->stream;
	const int64_t n = csr->n, m = csr->m, vsize = n + 2;
	const unsigned big_grid = (unsigned)csr->ctx->sm_count * 16;
	int32_t *ref_off;
	PGQ_TRY(ref_offsets(csr, ws, s, &ref_off, &st->kernel_launches));
	// the in-CSC in original ids, in-lists by ascending source: the edges in reference order, stably sorted by target
	int32_t *key_a, *key_b, *val_a, *val_b, *key_res, *in_src, *in_off, *scan_tmp, *dflag;
	const size_t mb = (size_t)std::max<int64_t>(m, 1) * sizeof(int32_t);
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_KEY_A, mb, (void **)&key_a));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_KEY_B, mb, (void **)&key_b));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_VAL_A, mb, (void **)&val_a));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_VAL_B, mb, (void **)&val_b));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_IN_OFF, (size_t)(vsize + 1) * sizeof(int32_t), (void **)&in_off));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_SCAN, pgq_scan_tmp_elems(vsize + 1) * sizeof(int32_t), (void **)&scan_tmp));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_DFLAG, (size_t)(vsize + 1) * sizeof(int32_t), (void **)&dflag));
	PGQ_CUDA(cudaMemsetAsync(in_off, 0, (size_t)(vsize + 1) * sizeof(int32_t), s));
	in_src = val_a;
	if (m > 0) {
		k_pr_ref_edges<<<an_grid(n * 32, 256, big_grid), 256, 0, s>>>(csr->out.off, csr->out.adj, csr->inv, n, ref_off,
		                                                               key_a, val_a);
		PGQ_CUDA(cudaGetLastError());
		PGQ_TRY(radix_sort_pairs(ws, key_a, key_b, val_a, val_b, m, bits_for(n), s, &key_res, &in_src));
		k_pr_histogram<<<an_grid(m, 256, big_grid), 256, 0, s>>>(key_res, m, in_off);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches += 2 + 2 * ((bits_for(n) + 4) / 5);
	}
	PGQ_TRY(pgq_scan_exclusive_i32(in_off, in_off, vsize + 1, scan_tmp, s));
	double *rank, *temp, *contrib, *dangling, *d_total;
	u64 *max_bits, *h_max;
	const size_t vb = (size_t)vsize * sizeof(double);
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_RANK, vb, (void **)&rank));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_TEMP, vb, (void **)&temp));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_CONTRIB, vb, (void **)&contrib));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_DANGLING, vb, (void **)&dangling));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PR_TOTAL, 256, (void **)&d_total));
	PGQ_TRY(pgq_ws_pinned(ws, 256, (void **)&h_max));
	max_bits = (u64 *)(d_total + 1);
	k_pr_init<<<an_grid(vsize + 1, 256, big_grid), 256, 0, s>>>(vsize, ref_off, rank, contrib, dflag);
	PGQ_CUDA(cudaGetLastError());
	PGQ_TRY(pgq_scan_exclusive_i32(dflag, dflag, vsize + 1, scan_tmp, s));
	k_pr_dangling_stage<<<an_grid(vsize, 256, big_grid), 256, 0, s>>>(vsize, ref_off, dflag, rank, dangling);
	PGQ_CUDA(cudaGetLastError());
	int32_t n_dangling = 0;
	PGQ_CUDA(cudaMemcpyAsync(&n_dangling, dflag + vsize, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	st->kernel_launches += 4;

	// the dangling fold runs on a second stream, concurrently with the pull
	cudaStream_t side = nullptr;
	cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr}; // fork, join, fold begin, fold end
	int rc = PGQ_OK;
	do {
		cudaError_t e = cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
		for (int i = 0; i < 4 && e == cudaSuccess; i++) {
			e = cudaEventCreateWithFlags(&ev[i], i < 2 ? cudaEventDisableTiming : cudaEventDefault);
		}
		if (e != cudaSuccess) {
			cudaGetLastError();
			rc = pgq_fail(PGQ_ERR_CUDA, "pagerank: stream / event creation failed: %s", cudaGetErrorString(e));
			break;
		}
		int64_t iters = 0;
		double fold_ms = 0.0;
		for (;;) {
			cudaMemsetAsync(max_bits, 0, sizeof(u64), s);
			cudaEventRecord(ev[0], s);
			cudaStreamWaitEvent(side, ev[0], 0);
			cudaEventRecord(ev[2], side);
			k_pr_dangling_fold<<<1, 32, 0, side>>>(dangling, n_dangling, d_total);
			cudaEventRecord(ev[3], side);
			cudaEventRecord(ev[1], side);
			k_pr_pull<<<an_grid(vsize * 32, 256, big_grid), 256, 0, s>>>(vsize, in_off, in_src, contrib, temp);
			cudaStreamWaitEvent(s, ev[1], 0);
			k_pr_update<<<an_grid(vsize, 256, big_grid), 256, 0, s>>>(vsize, ref_off, rank, temp, contrib, dflag,
			                                                          dangling, d_total, max_bits);
			cudaMemcpyAsync(h_max, max_bits, sizeof(u64), cudaMemcpyDeviceToHost, s);
			e = cudaStreamSynchronize(s);
			if (e == cudaSuccess) {
				e = cudaGetLastError();
			}
			if (e != cudaSuccess) {
				rc = pgq_fail(PGQ_ERR_CUDA, "pagerank iteration failed: %s", cudaGetErrorString(e));
				break;
			}
			float ms = 0.0f;
			cudaEventElapsedTime(&ms, ev[2], ev[3]);
			fold_ms += ms;
			st->kernel_launches += 3;
			std::swap(rank, temp);
			iters++;
			double max_delta;
			memcpy(&max_delta, h_max, sizeof(double));
			if (max_delta < 1e-6) { // pagerank.cpp:74-78
				break;
			}
		}
		if (rc != PGQ_OK) {
			break;
		}
		csr->pr_rank.resize((size_t)vsize);
		if (cudaMemcpyAsync(csr->pr_rank.data(), rank, vb, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
		    cudaStreamSynchronize(s) != cudaSuccess) {
			cudaGetLastError();
			csr->pr_rank.clear();
			rc = pgq_fail(PGQ_ERR_CUDA, "pagerank: copying the ranks back failed");
			break;
		}
		st->d2h_bytes += (int64_t)vb;
		st->levels = iters;
		st->expand_ms = fold_ms;
		csr->pr_iters = iters;
		csr->pr_done = true;
	} while (0);
	if (side) {
		cudaStreamSynchronize(side);
		cudaStreamDestroy(side);
	}
	for (cudaEvent_t x : ev) {
		if (x) {
			cudaEventDestroy(x);
		}
	}
	return rc;
}

// =================================================================================================================
// weakly_connected_component
// =================================================================================================================
// every out-edge as (a = source, b = target, k = reference CSR position), original ids, in internal order
__global__ void k_wcc_edges(const int32_t *__restrict__ off, const int32_t *__restrict__ adj,
                            const int32_t *__restrict__ inv, int64_t n, const int32_t *__restrict__ ref_off,
                            int32_t *__restrict__ ea, int32_t *__restrict__ eb, int32_t *__restrict__ ek) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t r = warp; r < n; r += nwarps) {
		const int32_t a = inv[r];
		const int b = off[r], len = off[r + 1] - b, base = ref_off[a];
		for (int j = lane; j < len; j += 32) {
			ea[b + j] = a;
			eb[b + j] = inv[adj[b + j]];
			ek[b + j] = base + j;
		}
	}
}

__global__ void k_wcc_init(int64_t n, int32_t *comp) {
	for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
		comp[v] = (int32_t)v;
	}
}

// best[c] = min over the edges with exactly one end in component c of (position << 32 | index in the edge list)
__global__ void k_wcc_min(int64_t count, const int32_t *__restrict__ ea, const int32_t *__restrict__ eb,
                          const int32_t *__restrict__ ek, const int32_t *__restrict__ comp, u64 *best) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
		const int32_t ca = comp[ea[i]], cb = comp[eb[i]];
		if (ca != cb) {
			const u64 key = ((u64)(uint32_t)ek[i] << 32) | (u64)i;
			atomicMin(&best[ca], key);
			atomicMin(&best[cb], key);
		}
	}
}

// Every component hooks under the other end of its least edge; when two components chose the same edge, the one
// with the smaller id stays a root.  Each chosen edge is recorded once, as (position, a, b).
__global__ void k_wcc_hook(int64_t n, const int32_t *__restrict__ ea, const int32_t *__restrict__ eb,
                           const int32_t *__restrict__ comp, const u64 *__restrict__ best, int32_t *hook,
                           int32_t *mk, int32_t *ma, int32_t *mb, int *n_merge) {
	for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (int64_t)gridDim.x * blockDim.x) {
		const u64 key = best[c];
		if (comp[c] != c || key == ~0ull) {
			hook[c] = (int32_t)c;
			continue;
		}
		const int64_t i = (int64_t)(key & 0xffffffffull);
		const int32_t a = ea[i], b = eb[i];
		const int32_t o = comp[a] == c ? comp[b] : comp[a];
		const bool mutual = best[o] == key;
		hook[c] = (mutual && c < o) ? (int32_t)c : o;
		if (!mutual || c < o) {
			const int slot = atomicAdd(n_merge, 1);
			mk[slot] = (int32_t)(key >> 32);
			ma[slot] = a;
			mb[slot] = b;
		}
	}
}

__global__ void k_wcc_jump(int64_t n, int32_t *hook, int *changed) {
	bool any = false;
	for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (int64_t)gridDim.x * blockDim.x) {
		const int32_t h = hook[c], hh = hook[h];
		if (h != hh) {
			hook[c] = hh;
			any = true;
		}
	}
	if (any) {
		*changed = 1;
	}
}

__global__ void k_wcc_relabel(int64_t n, int32_t *comp, const int32_t *__restrict__ hook) {
	for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
		comp[v] = hook[comp[v]];
	}
}

// keeps the edges whose ends lie in different components (order does not matter: the position travels along)
__global__ void k_wcc_compact(int64_t count, const int32_t *__restrict__ ea, const int32_t *__restrict__ eb,
                              const int32_t *__restrict__ ek, const int32_t *__restrict__ comp, int32_t *oa,
                              int32_t *ob, int32_t *ok, int *out_count) {
	const int lane = threadIdx.x & 31;
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < count; base += stride) {
		const int64_t i = base + threadIdx.x;
		const bool keep = i < count && comp[ea[i]] != comp[eb[i]];
		const uint32_t ball = __ballot_sync(AN_FULL, keep);
		int slot = 0;
		if (lane == 0 && ball) {
			slot = atomicAdd(out_count, __popc(ball));
		}
		slot = __shfl_sync(AN_FULL, slot, 0) + __popc(ball & ((1u << lane) - 1));
		if (keep) {
			oa[slot] = ea[i];
			ob[slot] = eb[i];
			ok[slot] = ek[i];
		}
	}
}

// FindTreeRoot, weakly_connected_component.cpp:14-24 (path halving)
static int64_t find_root(std::vector<int64_t> &forest, int64_t x) {
	while (forest[x] != x) {
		forest[x] = forest[forest[x]];
		x = forest[x];
	}
	return x;
}

// Finds the merge edges (Boruvka on the device), replays Link over them in position order on the host and keeps the
// label of all vsize entries in csr->wcc_label (called under csr->mu).
static int wcc_compute(pgq_csr *csr, Workspace *ws, pgq_stats *st) {
	cudaStream_t s = ws->stream;
	const int64_t n = csr->n, m = csr->m, vsize = n + 2;
	const unsigned big_grid = (unsigned)csr->ctx->sm_count * 16;
	std::vector<int32_t> h_a, h_b, h_order;
	int n_merge = 0;
	if (m > 0 && n > 0) {
		int32_t *ref_off;
		PGQ_TRY(ref_offsets(csr, ws, s, &ref_off, &st->kernel_launches));
		int32_t *e[6], *comp, *hook, *mk, *ma, *mb, *key_b, *idx_a, *idx_b, *key_res, *idx_res;
		const size_t mb_bytes = (size_t)m * sizeof(int32_t), nb = (size_t)(n + 1) * sizeof(int32_t);
		for (int i = 0; i < 6; i++) {
			PGQ_TRY(pgq_ws_reserve(ws, (WsSlot)(WS_WCC_EDGES + i), mb_bytes, (void **)&e[i]));
		}
		u64 *best;
		int *flags, *h_flags;
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_COMP, nb, (void **)&comp));
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_HOOK, nb, (void **)&hook));
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_BEST, (size_t)n * sizeof(u64), (void **)&best));
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_MERGE_POS, nb, (void **)&mk));
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_MERGE_A, nb, (void **)&ma));
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_MERGE_B, nb, (void **)&mb));
		PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_FLAGS, 256, (void **)&flags)); // [0] merges, [1] jump changed, [2] edges kept
		PGQ_TRY(pgq_ws_pinned(ws, 256, (void **)&h_flags));
		k_wcc_edges<<<an_grid(n * 32, 256, big_grid), 256, 0, s>>>(csr->out.off, csr->out.adj, csr->inv, n, ref_off, e[0],
		                                                            e[1], e[2]);
		k_wcc_init<<<an_grid(n, 256, big_grid), 256, 0, s>>>(n, comp);
		PGQ_CUDA(cudaMemsetAsync(flags, 0, 4 * sizeof(int), s));
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches += 2;
		int32_t **cur = e, **nxt = e + 3;
		int64_t count = m;
		while (count > 0) {
			PGQ_CUDA(cudaMemsetAsync(best, 0xff, (size_t)n * sizeof(u64), s));
			k_wcc_min<<<an_grid(count, 256, big_grid), 256, 0, s>>>(count, cur[0], cur[1], cur[2], comp, best);
			k_wcc_hook<<<an_grid(n, 256, big_grid), 256, 0, s>>>(n, cur[0], cur[1], comp, best, hook, mk, ma, mb, flags);
			st->kernel_launches += 2;
			for (;;) {
				PGQ_CUDA(cudaMemsetAsync(flags + 1, 0, sizeof(int), s));
				k_wcc_jump<<<an_grid(n, 256, big_grid), 256, 0, s>>>(n, hook, flags + 1);
				PGQ_CUDA(cudaMemcpyAsync(h_flags, flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
				PGQ_CUDA(cudaStreamSynchronize(s));
				st->kernel_launches++;
				if (!h_flags[1]) {
					break;
				}
			}
			k_wcc_relabel<<<an_grid(n, 256, big_grid), 256, 0, s>>>(n, comp, hook);
			PGQ_CUDA(cudaMemsetAsync(flags + 2, 0, sizeof(int), s));
			k_wcc_compact<<<an_grid(count, 256, big_grid), 256, 0, s>>>(count, cur[0], cur[1], cur[2], comp, nxt[0], nxt[1],
			                                                             nxt[2], flags + 2);
			PGQ_CUDA(cudaMemcpyAsync(h_flags + 2, flags + 2, sizeof(int), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			PGQ_CUDA(cudaGetLastError());
			st->kernel_launches += 2;
			st->levels++;
			count = h_flags[2];
			std::swap(cur, nxt);
		}
		n_merge = h_flags[0];
		if (n_merge > 0) {
			// the merge positions in ascending order (a stable radix sort of (position, index))
			PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_SORT_KEY, (size_t)n_merge * sizeof(int32_t), (void **)&key_b));
			PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_SORT_IDX_A, (size_t)n_merge * sizeof(int32_t), (void **)&idx_a));
			PGQ_TRY(pgq_ws_reserve(ws, WS_WCC_SORT_IDX_B, (size_t)n_merge * sizeof(int32_t), (void **)&idx_b));
			k_wcc_init<<<an_grid(n_merge, 256, big_grid), 256, 0, s>>>(n_merge, idx_a);
			PGQ_CUDA(cudaGetLastError());
			PGQ_TRY(radix_sort_pairs(ws, mk, key_b, idx_a, idx_b, n_merge, bits_for(m), s, &key_res, &idx_res));
			st->kernel_launches += 1 + 2 * ((bits_for(m) + 4) / 5);
			h_a.resize((size_t)n_merge);
			h_b.resize((size_t)n_merge);
			h_order.resize((size_t)n_merge);
			const size_t bytes = (size_t)n_merge * sizeof(int32_t);
			PGQ_CUDA(cudaMemcpyAsync(h_order.data(), idx_res, bytes, cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaMemcpyAsync(h_a.data(), ma, bytes, cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaMemcpyAsync(h_b.data(), mb, bytes, cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st->d2h_bytes += 3 * (int64_t)bytes;
		}
	}
	// Link (weakly_connected_component.cpp:26-35) over the merge edges in position order; forest[n + 1] = 0 is the
	// value-initialised entry the reference's loop never sets (l.57-60)
	std::vector<int64_t> forest((size_t)vsize);
	for (int64_t i = 0; i < vsize - 1; i++) {
		forest[i] = i;
	}
	forest[vsize - 1] = 0;
	for (int i = 0; i < n_merge; i++) {
		const int32_t j = h_order[i];
		const int64_t ra = find_root(forest, h_a[j]), rb = find_root(forest, h_b[j]);
		if (ra != rb) {
			forest[ra] = rb;
		}
	}
	csr->wcc_label.resize((size_t)vsize);
	for (int64_t v = 0; v < vsize; v++) {
		csr->wcc_label[v] = find_root(forest, v);
	}
	csr->wcc_done = true;
	return PGQ_OK;
}

// =================================================================================================================
// entry points of the cached functions
// =================================================================================================================
// Runs `compute` once per CSR under its mutex (concurrent first callers wait for the first one).
template <typename F>
static int ensure_cached(pgq_csr *csr, bool pgq_csr::*done, pgq_stats *st, F compute) {
	std::lock_guard<std::mutex> g(csr->mu);
	if (csr->*done) {
		return PGQ_OK;
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard wg(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &wg.ws));
	Workspace *ws = wg.ws;
	cudaEventRecord(ws->ev_begin, ws->stream);
	PGQ_TRY(compute(csr, ws, st));
	cudaEventRecord(ws->ev_end, ws->stream);
	cudaError_t e = cudaStreamSynchronize(ws->stream);
	if (e != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) {
		return pgq_fail(PGQ_ERR_CUDA, "analytics computation failed: %s", cudaGetErrorString(e));
	}
	wg.settled = true;
	float ms = 0.0f;
	cudaEventElapsedTime(&ms, ws->ev_begin, ws->ev_end);
	st->total_ms = ms;
	cudaGetLastError();
	return PGQ_OK;
}

static int check_cached_call(pgq_csr *csr, int64_t p, const int64_t *src, const void *out, const uint8_t *out_valid) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (p < 0 || (p > 0 && (!src || !out || !out_valid))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	return PGQ_OK;
}

extern "C" int pgq_pagerank(pgq_csr *csr, int64_t p, const int64_t *src, const uint8_t *src_valid, double *out,
                            uint8_t *out_valid, int64_t *iterations, pgq_stats *stats) {
	PGQ_TRY(check_cached_call(csr, p, src, out, out_valid));
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	PGQ_TRY(ensure_cached(csr, &pgq_csr::pr_done, &st, pagerank_compute));
	const int64_t vsize = csr->n + 2;
	for (int64_t r = 0; r < p; r++) {
		const bool ok = (!src_valid || src_valid[r]) && src[r] >= 0 && src[r] < vsize; // pagerank.cpp:96-103
		out[r] = ok ? csr->pr_rank[src[r]] : 0.0;
		out_valid[r] = ok;
	}
	if (iterations) {
		*iterations = csr->pr_iters;
	}
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_weakly_connected_component(pgq_csr *csr, int64_t p, const int64_t *src, const uint8_t *src_valid,
                                              int64_t *out, uint8_t *out_valid, pgq_stats *stats) {
	PGQ_TRY(check_cached_call(csr, p, src, out, out_valid));
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	PGQ_TRY(ensure_cached(csr, &pgq_csr::wcc_done, &st, wcc_compute));
	const int64_t vsize = csr->n + 2;
	for (int64_t r = 0; r < p; r++) {
		const bool ok = (!src_valid || src_valid[r]) && src[r] >= 0 && src[r] < vsize; // l.89-97
		out[r] = ok ? csr->wcc_label[src[r]] : 0;
		out_valid[r] = ok;
	}
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}
