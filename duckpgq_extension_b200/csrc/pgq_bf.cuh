// pgq_bf.cuh -- what the Bellman-Ford files share (pgq_cheapest.cu, pgq_cheapest_k.cu): the order-preserving keys of
// the distances, the "unreachable" sentinel, the distance fill and the dirty-vertex sweep, which cheapest_k_paths runs
// over the edges its spur searches admit (pgq_cheapest.cu's top describes the sweep).
#pragma once

#include "pgq_internal.h"
#include "pgq_tile.cuh"

#define BF_INF_I64 (0x7fffffffffffffffLL / 2)
#define BF_INF_F64 (1.7976931348623157e308 / 2)

// doubles are kept as order-preserving unsigned keys so that atomicMin works on them
__device__ __forceinline__ u64 f64_key(double d) {
	const u64 b = (u64)__double_as_longlong(d);
	return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_f64(u64 k) {
	const u64 b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
	return __longlong_as_double((long long)b);
}

template <bool F64>
__global__ void k_bf_init(int64_t count, u64 *dist) {
	const u64 inf = F64 ? f64_key(1.7976931348623157e308 / 2) : (u64)BF_INF_I64;
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
		dist[i] = inf;
	}
}

// The edge filter of k_bf_sweep: every edge relaxes, for every lane, with the reference's unguarded sum.  A filter
// answers whether the edge at out-CSR position e into u may relax lane l from the distance key dk over weight bits w.
struct BfAllEdges {
	__device__ __forceinline__ bool edge(int64_t e, int u, int l, u64 dk, int64_t w) const {
		return true;
	}
};

// One sweep: a warp per dirty vertex relaxes all of its out-edges for all lanes (UpdateLanes, l.38-50) that `keep`
// admits (every edge by default).
template <bool F64, class EdgeFilter = BfAllEdges>
__global__ void __launch_bounds__(256) k_bf_sweep(int64_t n, int L, const int32_t *__restrict__ off,
                                                  const int32_t *__restrict__ adj, const int64_t *__restrict__ w_bits,
                                                  u64 *dist, uint32_t *dirty, int *changed,
                                                  const EdgeFilter keep = EdgeFilter()) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	bool any = false;
	for (int64_t v = warp; v < n; v += nwarps) {
		const uint32_t bit = 1u << (v & 31);
		if (!(dirty[v >> 5] & bit)) {
			continue;
		}
		if (lane == 0) {
			atomicAnd(&dirty[v >> 5], ~bit); // cleared BEFORE the distances are read: a later improvement marks it again
		}
		__syncwarp();
		__threadfence();
		const int e0 = off[v], e1 = off[v + 1];
		for (int g = 0; g < L; g += 32) {
			const u64 dk = *reinterpret_cast<volatile u64 *>(&dist[v * L + g + lane]);
			for (int e = e0; e < e1; e++) {
				const int u = adj[e];
				u64 nk;
				bool is_nan = false;
				if (F64) {
					const double c = key_f64(dk) + __longlong_as_double(w_bits[e]);
					is_nan = c != c; // new_dist < n_dist is false for a NaN (UpdateOneLane l.31)
					nk = f64_key(c);
				} else {
					nk = dk + (u64)w_bits[e]; // (wraps: a filter that rejects the edge may reject an overflowed sum)
				}
				u64 *slot = &dist[(int64_t)u * L + g + lane];
				bool better;
				if (F64) {
					better = !is_nan && keep.edge(e, u, g + lane, dk, w_bits[e]) &&
					         nk < *reinterpret_cast<volatile u64 *>(slot) && nk < atomicMin(slot, nk);
				} else {
					better = keep.edge(e, u, g + lane, dk, w_bits[e]) &&
					         (long long)nk < *reinterpret_cast<volatile long long *>(slot) &&
					         (long long)nk < atomicMin(reinterpret_cast<long long *>(slot), (long long)nk);
				}
				if (__any_sync(FULL_MASK, better)) {
					if (lane == 0) {
						__threadfence();
						atomicOr(&dirty[u >> 5], 1u << (u & 31));
					}
					any = true;
				}
			}
		}
	}
	if (any && lane == 0) {
		*changed = 1;
	}
}
