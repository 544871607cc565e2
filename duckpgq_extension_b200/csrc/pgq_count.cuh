// pgq_count.cuh -- what the path-counting files share (pgq_allshortest.cu, pgq_kshortest.cu, pgq_cheapest.cu):
// saturating counts, the step-ordered in-lists, and the walk engine (pgq_kshortest.cu's top describes it): its backward
// reach, layered walk counts and unranking kernels, and the host driver that runs them, for shortest_k_paths over every
// edge and for all_cheapest_paths over the tight edges of each lane.
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

// The walk kernels' counters: [0] a backward level added a bit; [1] lanes still counting; [2] a lane needs a walk longer
// than KS_WALK_MAX
enum { KS_CHANGED = 0, KS_ACTIVE = 1, KS_TOO_LONG = 2 };

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

// ---- the walk engine's host driver ----------------------------------------------------------------------------------
// A call's walk engine: its CSR, workspace and stats, the in-lists its kernels walk (csr->in.adj, or the step lists'
// parents), its staged columns and step lists, and its device buffers in the WS_KS_* slots (pgq_internal.h); walks and
// elem_total count the walks placed so far and their elements.  `what` names the walks in the call's messages.
struct Walk {
	pgq_csr *csr;
	Workspace *ws;
	pgq_stats *st;
	const char *what;
	const int32_t *in_list;
	const int64_t *src, *dst;
	const u64 *step_key;
	const int32_t *step_pos;
	const int32_t *lane_row;
	int32_t *psrc, *pdst, *glane, *gsrc;
	u64 *reach, *front, *next, *om_a, *om_b, *total, *act, *ctr;
	uint32_t *alive;
	int64_t *npaths, *elems_row, *last, *first, *elem_off, *walk_off, *elems;
	u64 walks, elem_total;
};

// reserve the engine's buffers: its per-row arrays for p rows; its per-lane buffers for `lanes` lane ids in batches W
// lanes wide (lane_row is the caller's)
int walk_reserve_rows(Walk &w, int64_t p);
int walk_reserve_lanes(Walk &w, int64_t lanes, int W);

// The backward reach of a batch, from the targets its caller seeded into reach and front: levels over the in-lists, each
// passing a lane's bits along the edges `keep` admits for it, until a level adds no bit.  cells = n x wd mask words.
template <class EdgeFilter>
int walk_reach(Walk &w, int wd, int64_t cells, const EdgeFilter &keep) {
	pgq_csr *csr = w.csr;
	cudaStream_t s = w.ws->stream;
	const int64_t m = csr->m;
	const int sms = csr->ctx->sm_count;
	u64 changed;
	for (;;) {
		PGQ_CUDA(cudaMemsetAsync(&w.ctr[KS_CHANGED], 0, sizeof(u64), s));
		if (m > 0) {
			k_ks_reach_level<<<grid_size((m + 255) / 256, (int64_t)sms * 16), 256, 0, s>>>(m, csr->n_ab, wd, csr->in.off,
			                                                                               w.in_list, w.front, w.reach,
			                                                                               w.next, keep);
			w.st->kernel_launches++;
		}
		k_ks_reach_update<<<grid_size((cells + 255) / 256, (int64_t)sms * 8), 256, 0, s>>>(cells, w.reach, w.front, w.next,
		                                                                                   w.ctr);
		PGQ_CUDA(cudaGetLastError());
		w.st->kernel_launches++;
		w.st->push_levels++;
		PGQ_CUDA(cudaMemcpyAsync(&changed, &w.ctr[KS_CHANGED], sizeof(u64), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		if (!changed) {
			return PGQ_OK;
		}
	}
}

// The counting pass of a batch of cnt lanes in layers L wide (psrc: the batch's sources): start() launches the caller's
// layer-0 kernel, which flags the lanes that count; then, while a lane counts, layer h = 1, 2, ... sums the edges `admit`
// admits (k_ks_omega) and step(h, cur) launches the caller's step kernel on it.  *layers counts the layers; a lane past
// KS_WALK_MAX fails the call with too_long.
template <class EdgeFilter, class Start, class Step>
int walk_count(Walk &w, int L, int cnt, int wd, const int32_t *psrc, const EdgeFilter &admit, const Start &start,
               const Step &step, int64_t *layers, const char *too_long) {
	pgq_csr *csr = w.csr;
	cudaStream_t s = w.ws->stream;
	const int64_t m = csr->m, n_ab = csr->n_ab;
	const size_t layer = (size_t)std::max<int64_t>(n_ab, 1) * L * sizeof(u64);
	const unsigned chunk_grid = grid_size((m + KS_CHUNK * 8 - 1) / (KS_CHUNK * 8), (int64_t)csr->ctx->sm_count * 16);
	u64 h_ctr[3];
	PGQ_CUDA(cudaMemsetAsync(w.ctr, 0, sizeof(h_ctr), s));
	start();
	PGQ_CUDA(cudaGetLastError());
	w.st->kernel_launches++;
	PGQ_CUDA(cudaMemcpyAsync(h_ctr, w.ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	u64 *prev = w.om_a, *cur = w.om_b;
	for (int h = 1; h_ctr[KS_ACTIVE] > 0; h++) {
		PGQ_CUDA(cudaMemsetAsync(cur, 0, layer, s));
		PGQ_CUDA(cudaMemsetAsync(&w.ctr[KS_ACTIVE], 0, sizeof(u64), s));
		if (m > 0) {
			k_ks_omega<<<chunk_grid, 256, 0, s>>>(h, m, n_ab, L, cnt, csr->in.off, w.in_list, psrc, prev, cur, w.reach,
			                                      w.act, wd, w.alive, admit);
			w.st->kernel_launches++;
		}
		step(h, cur);
		PGQ_CUDA(cudaGetLastError());
		w.st->kernel_launches++;
		(*layers)++;
		PGQ_CUDA(cudaMemcpyAsync(h_ctr, w.ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		if (h_ctr[KS_TOO_LONG]) {
			return pgq_fail(PGQ_ERR_UNSUPPORTED, "%s %d edges", too_long, KS_WALK_MAX);
		}
		std::swap(prev, cur);
	}
	return PGQ_OK;
}

// Places the walks of rows [lo, hi) behind the walks placed so far: checks that the call's walks and their elements stay
// addressable (h_np, h_el: host copies of the rows' walk and element counts), scans the rows' first element and first
// walk from the running totals (valid = the row has a walk), and grows the offset and element buffers to hold them.
int walk_offsets(Walk &w, int64_t lo, int64_t hi, const int64_t *h_np, const int64_t *h_el, uint8_t *valid);

// A lane whose row has walks, the longest of them `last` edges long
struct WalkLane {
	int32_t lane;
	int64_t row, last;
};

// The storing pass and the unranking of `lanes`: packed greedily in order into groups of at most cap lanes whose layers,
// (H + 1) x n_ab x lanes x 8 B with H the group's longest walk, fit the budget; each group recomputes its layers, every
// one kept, and unranks its walks into the offsets walk_offsets placed.  filter_for(glane) is the edge filter of a group
// whose lane j is lane glane[j] of the engine.
template <class FilterFor>
int walk_store(Walk &w, const std::vector<WalkLane> &lanes, int cap, int64_t budget, const FilterFor &filter_for) {
	pgq_csr *csr = w.csr;
	cudaStream_t s = w.ws->stream;
	const int64_t n = csr->n, m = csr->m, n_ab = csr->n_ab;
	const int sms = csr->ctx->sm_count;
	const unsigned chunk_grid = grid_size((m + KS_CHUNK * 8 - 1) / (KS_CHUNK * 8), (int64_t)sms * 16);
	std::vector<int32_t> grp;
	int64_t grp_h = 0;
	auto layer_bytes = [&](int64_t h, int64_t rows) { return (double)(h + 1) * (double)n_ab * (double)rows * 8.0; };
	auto run_group = [&]() -> int {
		const int ng = (int)grp.size();
		if (ng == 0) {
			return PGQ_OK;
		}
		u64 *layers;
		PGQ_TRY(pgq_ws_reserve(w.ws, WS_KS_LAYERS, (size_t)std::max<int64_t>(grp_h, 1) * n_ab * ng * sizeof(u64),
		                       (void **)&layers));
		PGQ_CUDA(cudaMemcpyAsync(w.glane, grp.data(), (size_t)ng * sizeof(int32_t), cudaMemcpyHostToDevice, s));
		k_ks_group_src<<<grid_size((ng + 255) / 256, 64), 256, 0, s>>>(ng, w.glane, w.psrc, w.gsrc);
		PGQ_CUDA(cudaGetLastError());
		w.st->kernel_launches++;
		w.st->h2d_bytes += ng * (int64_t)sizeof(int32_t);
		if (grp_h > 0) {
			PGQ_CUDA(cudaMemsetAsync(layers, 0, (size_t)grp_h * n_ab * ng * sizeof(u64), s));
		}
		const auto admit = filter_for(w.glane);
		for (int64_t h = 1; h <= grp_h && m > 0; h++) {
			u64 *lcur = layers + (h - 1) * n_ab * ng;
			const u64 *lprev = h >= 2 ? layers + (h - 2) * n_ab * ng : nullptr;
			k_ks_omega<<<chunk_grid, 256, 0, s>>>((int)h, m, n_ab, ng, ng, csr->in.off, w.in_list, w.gsrc, lprev, lcur,
			                                      nullptr, nullptr, 0, nullptr, admit);
			w.st->kernel_launches++;
		}
		k_ks_unrank<<<grid_size(ng, (int64_t)sms * 16), 256, 0, s>>>(
		    ng, ng, n, n_ab, w.glane, w.lane_row, w.psrc, w.pdst, w.src, w.dst, layers, csr->in.off, w.step_key,
		    w.step_pos, csr->perm, csr->edge_ids, w.npaths, w.last, w.first, w.elem_off, w.walk_off, w.elems, admit);
		PGQ_CUDA(cudaGetLastError());
		w.st->kernel_launches++;
		// (the next group reuses the group buffers)
		PGQ_CUDA(cudaStreamSynchronize(s));
		grp.clear();
		grp_h = 0;
		return PGQ_OK;
	};
	for (const WalkLane &ln : lanes) {
		if (layer_bytes(ln.last, 1) > (double)budget) {
			return pgq_fail(PGQ_ERR_UNSUPPORTED, "the %s of row %lld need %.0f bytes of count layers, over the budget of "
			                "%lld", w.what, (long long)ln.row, layer_bytes(ln.last, 1), (long long)budget);
		}
		const int64_t gh = std::max(grp_h, ln.last);
		if (!grp.empty() && ((int64_t)grp.size() == cap || layer_bytes(gh, (int64_t)grp.size() + 1) > (double)budget)) {
			PGQ_TRY(run_group());
		}
		grp.push_back(ln.lane);
		grp_h = std::max(grp_h, ln.last);
	}
	return run_group();
}

// Ends the call's timing once the work queued so far (e: the first error in queueing it) has finished, and marks the
// call settled; `what` names the results being copied back in the error
int walk_end(WsGuard &g, pgq_stats *st, const char *what, cudaError_t e = cudaSuccess);

// Copies the placed walks back as the call's lists (offsets closed by the element total, elements), the rows' first walk
// and validity (d_valid, p rows), and ends the call's timing.  d2h_bytes counts the lists and the validity; the caller
// counts the per-row arrays it copies.
int walk_lists(Walk &w, WsGuard &g, int64_t p, const uint8_t *d_valid, int64_t *out_first_path, uint8_t *out_valid,
               int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths);

// The lists of a call without rows: offsets {0} and no elements (nor costs, with out_costs), as host allocations
int empty_lists(int64_t **out_path_offsets, int64_t **out_elems, void **out_costs = nullptr);
