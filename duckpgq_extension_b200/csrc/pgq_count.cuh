// pgq_count.cuh -- what the path-counting files share (pgq_allshortest.cu, pgq_kshortest.cu, pgq_cheapest.cu):
// saturating counts, the step-ordered in-lists, and the walk engine's backward reach, layered walk counts and unranking
// (pgq_kshortest.cu's top describes them), which all_cheapest_paths runs over the tight edges of each lane.
#pragma once

#include "pgq_internal.h"
#include "pgq_tile.cuh"

#define AS_MAX 0x7fffffffffffffffull

__device__ __forceinline__ u64 sat_add(u64 a, u64 b) { // a, b <= INT64_MAX
	const u64 s = a + b;
	return s > AS_MAX ? AS_MAX : s;
}

// *a = sat_add(*a, v); returns the old value
__device__ __forceinline__ u64 atomic_sat_add(u64 *a, u64 v) {
	u64 old = *reinterpret_cast<volatile u64 *>(a), assumed;
	do {
		assumed = old;
		old = atomicCAS(a, assumed, sat_add(assumed, v));
	} while (old != assumed);
	return old;
}

// The step lists of the CSR into the workspace (WS_AS_STEP_*; pgq_allshortest.cu): every out-edge v -> u keyed
// u * n + (original id of v) with its out-CSR position as value, stably sorted, so that u's in-edges in step order --
// the parent's ORIGINAL id, then the edge's position in the parent's adjacency -- sit at [in_off[u], in_off[u + 1]).
int build_step_lists(pgq_csr *csr, Workspace *ws, cudaStream_t s, const u64 **keys, const int32_t **pos,
                     int64_t *launches);

// shortest_k_paths' argument checks, shared by every path mode: the outputs are cleared first, then null and negative
// arguments, k < 1, lanes, the pair count, an unfinalised CSR and shard_count, in that order
int ks_check_call(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const pgq_options *opts, int64_t k,
                  const int64_t *out_npaths, const int64_t *out_first_path, const uint8_t *out_valid,
                  int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths);

// shortest_k_groups in WALK mode (pgq_kshortest.cu), over arguments pgq_shortest_k_groups has checked
int kg_walk(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
            const uint8_t *dst_valid, const pgq_options *opts, int64_t k, int64_t max_paths, int64_t *out_count,
            int64_t *out_ngroups, int64_t *out_last_len, uint8_t *out_complete, int64_t *out_npaths,
            int64_t *out_first_path, uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
            int64_t *out_total_paths, pgq_stats *stats);

#define KS_WALK_MAX 65533   // the longest walk a result may hold (all_shortest_paths' depth limit)

// pgq_kshortest.cu's fold of a backward level (the new bits become the frontier and join the reach; ctr[0] = 1 when
// a bit was new) and the sources of a storing group's lanes (gsrc[j] = psrc[glane[j]])
__global__ void k_ks_reach_update(int64_t cells, u64 *reach, u64 *front, u64 *next, u64 *ctr);
__global__ void k_ks_group_src(int ng, const int32_t *__restrict__ glane, const int32_t *__restrict__ psrc,
                               int32_t *gsrc);

// the storing pass's layer budget: 4 GiB, or PGQ_B200_KSP_LAYER_BUDGET bytes (tests force regrouping with it)
int layer_budget(int64_t *out);

// The edge filter of the walk kernels below: every edge, for every lane.  A filter answers for the edge at position e of
// the in-lists the kernel walks, from -> to (internal ids), whether lane l admits it (edge), and which of the 64 lanes
// of word j in `cand` do (lanes).
struct AllEdges {
	__device__ __forceinline__ bool edge(int64_t e, int64_t from, int64_t to, int l) const {
		return true;
	}
	__device__ __forceinline__ u64 lanes(int64_t e, int64_t from, int64_t to, int j, u64 cand) const {
		return cand;
	}
};

#define KS_CHUNK 128        // in-CSC positions per warp of k_ks_omega
__device__ __forceinline__ u64 sat_mul_len(u64 c, int64_t len) { // c <= INT64_MAX, len >= 1
	return c > AS_MAX / (u64)len ? AS_MAX : c * (u64)len;
}

// the largest row u < n_ab with in_off[u] <= e (rows below n_ab have in-edges, so their offsets rise strictly)
__device__ __forceinline__ int64_t ks_row_of(const int32_t *__restrict__ in_off, int64_t n_ab, int64_t e) {
	int64_t lo = 0, hi = n_ab - 1;
	while (lo < hi) {
		const int64_t mid = (lo + hi + 1) >> 1;
		if (in_off[mid] <= e) {
			lo = mid;
		} else {
			hi = mid - 1;
		}
	}
	return lo;
}

// one backward level: every in-edge u -> v of a frontier vertex v passes v's new lanes on to u.  A thread per in-CSC
// position; a warp finds the row of its first position by bisection and each thread walks on from there.  `keep` passes
// a lane's bit along the edges it admits for that lane (every edge by default).
template <class EdgeFilter = AllEdges>
__global__ void __launch_bounds__(256) k_ks_reach_level(int64_t m, int64_t n_ab, int wd, const int32_t *__restrict__ in_off,
                                                        const int32_t *__restrict__ in_adj, const u64 *__restrict__ front,
                                                        const u64 *__restrict__ reach, u64 *next,
                                                        const EdgeFilter keep = EdgeFilter()) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t base = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; base < m; base += nwarps * 32) {
		int64_t v = ks_row_of(in_off, n_ab, base);
		const int64_t e = base + lane;
		if (e >= m) {
			continue;
		}
		while (in_off[v + 1] <= e) {
			v++;
		}
		const int64_t u = in_adj[e];
		for (int j = 0; j < wd; j++) {
			const u64 f = front[v * wd + j];
			if (f) {
				const u64 nb = keep.lanes(e, u, v, j, f & ~reach[u * wd + j]);
				if (nb) {
					atomicOr(&next[u * wd + j], nb);
				}
			}
		}
	}
}

// Layer h of w over L lanes (see the top).  h == 1 counts the edges from each lane's source (lane_src, nl real lanes);
// reach / act (nullable) restrict lane l to the rows of B(t_l) while it counts, and alive (nullable) flags each lane
// with a non-zero w_h; `admit` sums only the in-edges it admits for the lane (every edge by default).  cur must be
// zero on entry.
template <class EdgeFilter = AllEdges>
__global__ void __launch_bounds__(256) k_ks_omega(int h, int64_t m, int64_t n_ab, int L, int nl,
                                                  const int32_t *__restrict__ in_off, const int32_t *__restrict__ in_adj,
                                                  const int32_t *__restrict__ lane_src, const u64 *__restrict__ prev,
                                                  u64 *cur, const u64 *__restrict__ reach, const u64 *__restrict__ act,
                                                  int wd, uint32_t *alive,
                                                  const EdgeFilter admit = EdgeFilter()) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	const int64_t nchunks = (m + KS_CHUNK - 1) / KS_CHUNK;
	for (int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < nchunks; c += nwarps) {
		const int64_t c0 = c * KS_CHUNK, c1 = min(c0 + KS_CHUNK, m);
		const int64_t u0 = ks_row_of(in_off, n_ab, c0);
		for (int g = 0; g < nl; g += 32) {
			const int l = g + lane;
			const bool on = l < nl;
			const int s = on ? lane_src[l] : -1;
			const bool counting = on && (!act || ((act[l >> 6] >> (l & 63)) & 1));
			int64_t u = u0, e = c0;
			while (e < c1) {
				const int64_t rs = in_off[u], re = in_off[u + 1], end = min(re, c1);
				const bool keep = counting && (!reach || ((reach[u * wd + (l >> 6)] >> (l & 63)) & 1));
				if (__any_sync(FULL_MASK, keep)) {
					u64 sum = 0;
					for (; e < end; e++) {
						const int64_t v = in_adj[e];
						if (keep && admit.edge(e, v, u, l)) {
							sum = sat_add(sum, h == 1 ? (v == s ? 1ull : 0ull) : (v < n_ab ? prev[v * L + l] : 0ull));
						}
					}
					if (keep && sum) {
						if (rs >= c0 && re <= c1) {
							cur[u * L + l] = sum;
						} else {
							atomic_sat_add(&cur[u * L + l], sum);
						}
						if (alive) {
							alive[l] = 1;
						}
					}
				}
				e = end;
				u++;
			}
		}
	}
}

// The walks of a group's rows: a block per row (grid-stride), a warp per walk (see the top).  layers[h - 1] is w_h of
// the group, [n_ab][Lg]; `admit` skips the steps it does not admit for the group's lane j (none by default).
template <class EdgeFilter = AllEdges>
__global__ void __launch_bounds__(256) k_ks_unrank(int ng, int Lg, int64_t n, int64_t n_ab,
                                                   const int32_t *__restrict__ glane, const int32_t *__restrict__ lane_row,
                                                   const int32_t *__restrict__ psrc, const int32_t *__restrict__ pdst,
                                                   const int64_t *__restrict__ src, const int64_t *__restrict__ dst,
                                                   const u64 *__restrict__ layers, const int32_t *__restrict__ in_off,
                                                   const u64 *__restrict__ step_key, const int32_t *__restrict__ step_pos,
                                                   const int32_t *__restrict__ perm, const int64_t *__restrict__ edge_ids,
                                                   const int64_t *__restrict__ npaths, const int64_t *__restrict__ last,
                                                   const int64_t *__restrict__ first, const int64_t *__restrict__ elem_off,
                                                   int64_t *walk_off, int64_t *elems,
                                                   const EdgeFilter admit = EdgeFilter()) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
	const int64_t layer_cells = n_ab * Lg;
	for (int j = blockIdx.x; j < ng; j += gridDim.x) {
		const int ln = glane[j];
		const int row = lane_row[ln];
		const int s = psrc[ln], t = pdst[ln];
		const int H = (int)last[row];
		const int64_t np = npaths[row];
		for (int64_t rank = warp; rank < np; rank += nw) {
			// the walk's length h, and the walks of its row before it of other lengths (count and elements)
			u64 carry_c = 0, carry_e = 0, before_c = 0, before_e = 0;
			int h = -1;
			for (int h0 = 0; h0 <= H && h < 0; h0 += 32) {
				const int hh = h0 + lane;
				u64 c = 0;
				if (hh <= H) {
					c = hh == 0 ? (s == t ? 1ull : 0ull)
					            : (t < n_ab ? layers[(int64_t)(hh - 1) * layer_cells + (int64_t)t * Lg + j] : 0ull);
				}
				u64 ic = c, ie = c ? sat_mul_len(c, 2 * (int64_t)hh + 1) : 0;
#pragma unroll
				for (int d = 1; d < 32; d <<= 1) {
					const u64 tc = __shfl_up_sync(FULL_MASK, ic, d), te = __shfl_up_sync(FULL_MASK, ie, d);
					if (lane >= d) {
						ic = sat_add(ic, tc);
						ie = sat_add(ie, te);
					}
				}
				const unsigned hit = __ballot_sync(FULL_MASK, sat_add(carry_c, ic) > (u64)rank);
				if (hit) {
					const int w = __ffs(hit) - 1;
					const u64 pc = __shfl_sync(FULL_MASK, ic, w > 0 ? w - 1 : 0);
					const u64 pe = __shfl_sync(FULL_MASK, ie, w > 0 ? w - 1 : 0);
					before_c = sat_add(carry_c, w > 0 ? pc : 0);
					before_e = sat_add(carry_e, w > 0 ? pe : 0);
					h = h0 + w;
				} else {
					carry_c = sat_add(carry_c, __shfl_sync(FULL_MASK, ic, 31));
					carry_e = sat_add(carry_e, __shfl_sync(FULL_MASK, ie, 31));
				}
			}
			if (h < 0) {
				break; // (cannot happen: the row's counts at t sum to at least npaths)
			}
			u64 r = (u64)rank - before_c;
			const int64_t len = 2 * (int64_t)h + 1;
			int64_t *out = elems + elem_off[row] + (int64_t)before_e + (int64_t)r * len;
			if (lane == 0) {
				walk_off[first[row] + rank] = out - elems;
				out[len - 1] = h == 0 ? src[row] : dst[row];
			}
			int cur = t;
			for (int k = h; k >= 1; k--) {
				const u64 *wl = k >= 2 ? layers + (int64_t)(k - 2) * layer_cells : nullptr;
				const int e1 = in_off[cur + 1];
				const u64 key0 = (u64)(uint32_t)cur * (u64)n;
				int pick_orig = -1, pick_pos = -1;
				for (int c = in_off[cur]; c < e1 && pick_pos < 0; c += 32) {
					const int e = c + lane;
					u64 wv = 0;
					int orig = 0, pos = 0;
					if (e < e1) {
						orig = (int)(step_key[e] - key0);
						pos = step_pos[e];
						const int par = perm[orig];
						if (admit.edge(e, par, cur, j)) {
							wv = k == 1 ? (par == s ? 1ull : 0ull) : (par < n_ab ? wl[(int64_t)par * Lg + j] : 0ull);
						}
					}
					u64 incl = wv;
#pragma unroll
					for (int d = 1; d < 32; d <<= 1) {
						const u64 tv = __shfl_up_sync(FULL_MASK, incl, d);
						if (lane >= d) {
							incl = sat_add(incl, tv);
						}
					}
					const unsigned hit = __ballot_sync(FULL_MASK, incl > r);
					if (hit) {
						const int w = __ffs(hit) - 1;
						const u64 before = __shfl_sync(FULL_MASK, incl, w > 0 ? w - 1 : 0);
						r -= w > 0 ? before : 0;
						pick_orig = __shfl_sync(FULL_MASK, orig, w);
						pick_pos = __shfl_sync(FULL_MASK, pos, w);
					} else {
						r -= __shfl_sync(FULL_MASK, incl, 31);
					}
				}
				if (pick_pos < 0) {
					break; // (cannot happen: w_k(cur) > r)
				}
				if (lane == 0) {
					out[2 * k - 1] = edge_ids[pick_pos];
					out[2 * k - 2] = pick_orig;
				}
				cur = perm[pick_orig];
			}
		}
	}
}

