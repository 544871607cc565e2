// pgq_kshortest.cu -- shortest_k_paths on the device CSR: the k shortest walks of a row (SQL/PGQ's SHORTEST k, which
// the reference parses and rejects).  No reference function.  sm_90a only.
//
// A lane is a row: the rows whose ids are both valid take lanes in input order, W per batch, with no source
// de-duplication, so that a row's answer never depends on the other rows of its batch.  Four phases:
//   * backward reach.  B(t), the vertices that reach the lane's target t (t included), as a W-bit mask per vertex: a
//     multi-lane BFS from the batch's targets over the in-CSC (k_ks_reach_level pushes each frontier bit from a vertex
//     to its in-neighbours, a thread per in-edge; k_ks_reach_update folds the level in), until a level adds no bit.
//     s outside B(t) makes the row NULL.  It has masks of its own: the BFS drivers' WS_SEEN / WS_VISIT_* keep their
//     known-zero record.
//   * counting pass.  w_h(u, l), the number of h-edge walks from the lane's source s to u, kept only for u in B(t):
//     w_0 is 1 at s (not stored), w_h(u) = the saturating sum of w_{h-1}(v) over the in-edges v -> u, and every vertex
//     of a level >= 1 has an in-edge, so layers have n_ab rows.  Two rolling layers [n_ab][L].  k_ks_omega pulls over
//     the in-CSC in chunks of KS_CHUNK edge positions, a warp per chunk and a thread per lane: a vertex whose in-list
//     lies inside one chunk is summed by one warp and stored, a longer one (an R-MAT hub) is split over the chunks it
//     spans, each adding its partial sum with atomic_sat_add.  Saturating addition of non-negative values is
//     associative, so neither the split nor the order changes a count.  A thread skips the rows outside its lane's
//     B(t) and the lanes that stopped.  k_ks_step then reads each lane's count at t, takes min(count, k - total)
//     walks of that length and stops the lane after the layer where its total reaches k or where w_h is zero on all
//     of B(t).  The second test is exact: a non-zero w at a vertex that reaches t means a longer walk to t exists.  It
//     is what ends the loop; without the restriction to B(t) a self-loop that s reaches but that does not reach t
//     would keep w alive forever.
//   * storing pass.  The rows with walks, packed greedily in lane order into groups of at most W rows whose layers
//     (H + 1) x n_ab x rows x 8 B fit the layer budget (H the group's longest walk), recompute w_1 .. w_H with the
//     same kernel, every layer kept.  No restriction there: H bounds the loop, and w is the same on B(t) with or
//     without it (every in-neighbour of a vertex of B(t) is in B(t)), which is all the unranking reads.
//   * unranking.  k_ks_unrank gives each listed walk a warp.  Walk r of a row finds its length h by a saturating
//     prefix sum of the row's counts at t over h = 0 .. H and its rank within that length, then walks back from t:
//     at node u with j steps left it scans u's step list (build_step_lists, shared with all_shortest_paths) with a
//     saturating prefix sum of w_{j-1}(parent) and takes the first edge whose prefix exceeds the rank, subtracting the
//     prefix before it.  Ranks stay exact under saturation by all_shortest_paths' argument: every rank is below k.
//     Element offsets: each row's element base is an exclusive scan of the rows' element counts (pgq_path_offsets),
//     and the walk adds the elements of the shorter walks of its row and of its rank's predecessors.
// shortest_k_groups in WALK mode runs the same four phases (ks_run) with k_kg_step in place of k_ks_step: k counts
// length groups, max_paths cuts the lists, and each row's rank bound is its listed count (DESIGN.md §3).
// k_ks_reach_level, k_ks_omega and k_ks_unrank live in pgq_count.cuh, templates over an edge filter, with the host
// driver that runs the phases (walk_*; its non-template parts are defined here): these calls take every edge
// (AllEdges), all_cheapest_paths (pgq_cheapest.cu) a lane's tight edges.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "pgq_count.cuh"
#include "pgq_tile.cuh"

#define KS_BUDGET ((int64_t)4 << 30)

// internal ids of the lanes' sources and targets
__global__ void k_ks_lanes(int64_t lanes, const int32_t *__restrict__ lane_row, const int64_t *__restrict__ src,
                           const int64_t *__restrict__ dst, const int32_t *__restrict__ perm, int32_t *psrc,
                           int32_t *pdst) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < lanes; i += (int64_t)gridDim.x * blockDim.x) {
		const int row = lane_row[i];
		psrc[i] = perm[src[row]];
		pdst[i] = perm[dst[row]];
	}
}

// level 0 of the backward reach: each lane's target
__global__ void k_ks_reach_seed(int cnt, int wd, const int32_t *__restrict__ pdst, u64 *reach, u64 *front) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		const int64_t cell = (int64_t)pdst[l] * wd + (l >> 6);
		atomicOr(&reach[cell], 1ull << (l & 63));
		atomicOr(&front[cell], 1ull << (l & 63));
	}
}

// folds a backward level in: the new bits become the frontier and join the reach
__global__ void k_ks_reach_update(int64_t cells, u64 *reach, u64 *front, u64 *next, u64 *ctr) {
	bool any = false;
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (int64_t)gridDim.x * blockDim.x) {
		const u64 nw = next[i] & ~reach[i];
		reach[i] |= nw;
		front[i] = nw;
		next[i] = 0;
		any |= nw != 0;
	}
	if (__any_sync(FULL_MASK, any) && (threadIdx.x & 31) == 0) {
		ctr[KS_CHANGED] = 1;
	}
}

// layer 0 of each lane: NULL when s is outside B(t); the walk [s] when s == t; the lane counts on while its total is
// below k
__global__ void k_ks_start(int cnt, int wd, int64_t k, const int32_t *__restrict__ lane_row,
                           const int32_t *__restrict__ psrc, const int32_t *__restrict__ pdst,
                           const u64 *__restrict__ reach, u64 *total, u64 *act, int64_t *npaths, int64_t *elems,
                           int64_t *last, u64 *ctr) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		const int row = lane_row[l];
		const int s = psrc[l], t = pdst[l];
		const bool in_b = (reach[(int64_t)s * wd + (l >> 6)] >> (l & 63)) & 1;
		const int64_t c0 = s == t ? 1 : 0;
		total[l] = c0;
		npaths[row] = c0;
		elems[row] = c0;
		last[row] = c0 ? 0 : -1;
		if (in_b && c0 < k) {
			atomicOr(&act[l >> 6], 1ull << (l & 63));
			atomicAdd(&ctr[KS_ACTIVE], 1ull);
		}
	}
}

// After layer h: each counting lane takes min(count at t, k - total) walks of h edges and stops when its total
// reaches k or w_h was zero on B(t)
__global__ void k_ks_step(int h, int cnt, int L, int64_t n_ab, int64_t k, const int32_t *__restrict__ lane_row,
                          const int32_t *__restrict__ pdst, const u64 *__restrict__ cur, uint32_t *alive, u64 *total,
                          u64 *act, int64_t *npaths, int64_t *elems, int64_t *last, u64 *ctr) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		if (!((act[l >> 6] >> (l & 63)) & 1)) {
			continue;
		}
		const int row = lane_row[l];
		const int t = pdst[l];
		const u64 c = t < n_ab ? cur[(int64_t)t * L + l] : 0;
		const u64 before = total[l];
		const u64 take = min(c, (u64)k - before);
		if (take) {
			total[l] = before + take;
			npaths[row] = (int64_t)(before + take);
			elems[row] = (int64_t)sat_add((u64)elems[row], sat_mul_len(take, 2 * (int64_t)h + 1));
			last[row] = h;
		}
		const bool stop = before + take >= (u64)k || !alive[l];
		alive[l] = 0;
		if (h > KS_WALK_MAX && (take || !stop)) {
			ctr[KS_TOO_LONG] = 1;
		}
		if (stop) {
			atomicAnd(&act[l >> 6], ~(1ull << (l & 63)));
		} else {
			atomicAdd(&ctr[KS_ACTIVE], 1ull);
		}
	}
}

// After layer h, for shortest_k_groups: a counting lane whose count c at t is non-zero finds length group h (lg counts
// the groups past h = 0, which s == t is), adds c to its saturating total and lists min(c, the room under max_paths)
// walks of h edges (all c for max_paths = 0); it stops after its k-th group or when w_h was zero on B(t)
__global__ void k_kg_step(int h, int cnt, int L, int64_t n_ab, int64_t k, int64_t max_paths,
                          const int32_t *__restrict__ lane_row, const int32_t *__restrict__ psrc,
                          const int32_t *__restrict__ pdst, const u64 *__restrict__ cur, uint32_t *alive, u64 *total,
                          int64_t *lg, u64 *act, int64_t *npaths, int64_t *elems, int64_t *last, u64 *ctr) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		if (!((act[l >> 6] >> (l & 63)) & 1)) {
			continue;
		}
		const int row = lane_row[l];
		const int t = pdst[l];
		const u64 c = t < n_ab ? cur[(int64_t)t * L + l] : 0;
		int64_t groups = lg[l] + (psrc[l] == t ? 1 : 0);
		if (c) {
			groups++;
			lg[l]++;
			total[l] = sat_add(total[l], c);
			last[row] = h;
			const u64 listed = (u64)npaths[row];
			const u64 take = max_paths ? min(c, (u64)max_paths - listed) : c;
			if (take) {
				npaths[row] = (int64_t)sat_add(listed, take);
				elems[row] = (int64_t)sat_add((u64)elems[row], sat_mul_len(take, 2 * (int64_t)h + 1));
			}
		}
		const bool stop = groups >= k || !alive[l];
		alive[l] = 0;
		if (h > KS_WALK_MAX && (c || !stop)) {
			ctr[KS_TOO_LONG] = 1;
		}
		if (stop) {
			atomicAnd(&act[l >> 6], ~(1ull << (l & 63)));
		} else {
			atomicAdd(&ctr[KS_ACTIVE], 1ull);
		}
	}
}

// the sources of a group's lanes
__global__ void k_ks_group_src(int ng, const int32_t *__restrict__ glane, const int32_t *__restrict__ psrc,
                               int32_t *gsrc) {
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < ng; j += gridDim.x * blockDim.x) {
		gsrc[j] = psrc[glane[j]];
	}
}

// ---- the walk engine's host driver (pgq_count.cuh) ----
static inline u64 sat_add_host(u64 a, u64 b) { // a, b <= INT64_MAX
	return a > AS_MAX - b ? AS_MAX : a + b;
}

int walk_reserve_rows(Walk &w, int64_t p) {
	Workspace *ws = w.ws;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_NPATHS, b8, (void **)&w.npaths));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_ROW_ELEMS, b8, (void **)&w.elems_row));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_LAST, b8, (void **)&w.last));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_FIRST, b8, (void **)&w.first));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_ELEM_OFF, b8, (void **)&w.elem_off));
	return PGQ_OK;
}

int walk_reserve_lanes(Walk &w, int64_t lanes, int W) {
	Workspace *ws = w.ws;
	const int wd = (W + 63) / 64;
	const size_t cells = (size_t)std::max<int64_t>(w.csr->n, 1) * wd;
	const size_t layer = (size_t)std::max<int64_t>(w.csr->n_ab, 1) * W;
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_PSRC, (size_t)lanes * sizeof(int32_t), (void **)&w.psrc));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_PDST, (size_t)lanes * sizeof(int32_t), (void **)&w.pdst));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_REACH, cells * sizeof(u64), (void **)&w.reach));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_FRONT, cells * sizeof(u64), (void **)&w.front));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_NEXT, cells * sizeof(u64), (void **)&w.next));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_OMEGA_A, layer * sizeof(u64), (void **)&w.om_a));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_OMEGA_B, layer * sizeof(u64), (void **)&w.om_b));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_TOTAL, (size_t)W * sizeof(u64), (void **)&w.total));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_ALIVE, (size_t)W * sizeof(uint32_t), (void **)&w.alive));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_ACTIVE, (size_t)wd * sizeof(u64), (void **)&w.act));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_COUNTERS, 256, (void **)&w.ctr));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_GROUP_LANE, (size_t)W * sizeof(int32_t), (void **)&w.glane));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_GROUP_SRC, (size_t)W * sizeof(int32_t), (void **)&w.gsrc));
	return PGQ_OK;
}

int walk_offsets(Walk &w, int64_t lo, int64_t hi, const int64_t *h_np, const int64_t *h_el, uint8_t *valid) {
	Workspace *ws = w.ws;
	cudaStream_t s = ws->stream;
	u64 walks = w.walks, elem_total = w.elem_total;
	for (int64_t i = 0; i < hi - lo; i++) {
		walks = sat_add_host(walks, (u64)h_np[i]);
		elem_total = sat_add_host(elem_total, (u64)h_el[i]);
	}
	if (elem_total > (AS_MAX / sizeof(int64_t)) || walks > (AS_MAX / sizeof(int64_t)) - 1) {
		return pgq_fail(PGQ_ERR_OOM, "the %s of one call hold too many elements (%llu)", w.what,
		                (unsigned long long)elem_total);
	}
	int64_t *d_total;
	PGQ_TRY(pgq_ws_reserve(ws, WS_KS_SCAN_TOTAL, sizeof(int64_t), (void **)&d_total));
	pgq_path_offsets((int64_t)w.elem_total, lo, hi, w.elem_off, w.elems_row, valid, d_total, s);
	pgq_path_offsets((int64_t)w.walks, lo, hi, w.first, w.npaths, valid, d_total, s); // (valid = a row has a walk)
	PGQ_CUDA(cudaGetLastError());
	w.st->kernel_launches += 2;
	// (grown, keeping what earlier batches placed; reserved at their size when there is nothing to keep)
	auto size = [&](WsSlot slot, u64 count, u64 keep, int64_t **out) {
		return keep ? pgq_ws_grow(ws, slot, (size_t)count * sizeof(int64_t), (size_t)keep * sizeof(int64_t), s, (void **)out)
		            : pgq_ws_reserve(ws, slot, (size_t)count * sizeof(int64_t), (void **)out);
	};
	PGQ_TRY(size(WS_KS_WALK_OFF, walks + 1, w.walks, &w.walk_off));
	PGQ_TRY(size(WS_KS_ELEMS, elem_total, w.elem_total, &w.elems));
	w.walks = walks;
	w.elem_total = elem_total;
	return PGQ_OK;
}

int walk_end(WsGuard &g, pgq_stats *st, const char *what, cudaError_t e) {
	Workspace *ws = g.ws;
	if (e == cudaSuccess) e = cudaEventRecord(ws->ev_end, ws->stream);
	if (e == cudaSuccess) e = cudaStreamSynchronize(ws->stream);
	float ms = 0.f;
	if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ws->ev_begin, ws->ev_end);
	g.settled = (e == cudaSuccess);
	if (e != cudaSuccess) {
		cudaGetLastError();
		return pgq_fail(PGQ_ERR_CUDA, "copying the %s back failed: %s", what, cudaGetErrorString(e));
	}
	st->total_ms = ms;
	return PGQ_OK;
}

int walk_lists(Walk &w, WsGuard &g, int64_t p, const uint8_t *d_valid, int64_t *out_first_path, uint8_t *out_valid,
               int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths) {
	cudaStream_t s = w.ws->stream;
	const u64 walks = w.walks, elem_total = w.elem_total;
	int64_t *h_off = (int64_t *)malloc((size_t)(walks + 1) * sizeof(int64_t));
	int64_t *h_elems = (int64_t *)malloc((size_t)std::max<u64>(elem_total, 1) * sizeof(int64_t));
	if (!h_off || !h_elems) {
		free(h_off);
		free(h_elems);
		return pgq_fail(PGQ_ERR_OOM, "host allocation of the %s' %llu elements failed", w.what,
		                (unsigned long long)elem_total);
	}
	cudaError_t e = cudaSuccess;
	if (walks > 0) e = cudaMemcpyAsync(h_off, w.walk_off, (size_t)walks * sizeof(int64_t), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess && elem_total > 0)
		e = cudaMemcpyAsync(h_elems, w.elems, (size_t)elem_total * sizeof(int64_t), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_first_path, w.first, (size_t)p * sizeof(int64_t), cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_valid, d_valid, (size_t)p, cudaMemcpyDeviceToHost, s);
	const int rc = walk_end(g, w.st, w.what, e);
	if (rc != PGQ_OK) {
		free(h_off);
		free(h_elems);
		return rc;
	}
	h_off[walks] = (int64_t)elem_total;
	w.st->d2h_bytes += p + (int64_t)(walks + elem_total) * (int64_t)sizeof(int64_t);
	*out_path_offsets = h_off;
	*out_elems = h_elems;
	*out_total_paths = (int64_t)walks;
	return PGQ_OK;
}

int empty_lists(int64_t **out_path_offsets, int64_t **out_elems, void **out_costs) {
	*out_path_offsets = (int64_t *)calloc(1, sizeof(int64_t));
	*out_elems = (int64_t *)malloc(sizeof(int64_t));
	if (out_costs) {
		*out_costs = malloc(sizeof(int64_t));
	}
	if (!*out_path_offsets || !*out_elems || (out_costs && !*out_costs)) {
		free(*out_path_offsets);
		free(*out_elems);
		*out_path_offsets = *out_elems = nullptr;
		if (out_costs) {
			free(*out_costs);
			*out_costs = nullptr;
		}
		return pgq_fail(PGQ_ERR_OOM, "host allocation failed");
	}
	return PGQ_OK;
}

// the layer budget of the storing pass: 4 GiB, or PGQ_B200_KSP_LAYER_BUDGET bytes (tests force regrouping with it)
int layer_budget(int64_t *out) {
	*out = KS_BUDGET;
	const char *env = getenv("PGQ_B200_KSP_LAYER_BUDGET");
	if (env && *env) {
		char *end = nullptr;
		const long long b = strtoll(env, &end, 10);
		if (*end || b <= 0) {
			return pgq_fail(PGQ_ERR_INVALID_ARG, "PGQ_B200_KSP_LAYER_BUDGET must be a positive byte count");
		}
		*out = b;
	}
	return PGQ_OK;
}

// the lane width: opts->lanes, or the widest of 512 .. 64 whose two counting layers fit 4 GiB, narrower while half of
// it would hold every lane
static int ks_lanes(const pgq_options *opts, int64_t n_ab, int64_t searches) {
	if (opts && opts->lanes) {
		return opts->lanes;
	}
	int w = 512;
	while (w > 64 && 2 * std::max<int64_t>(n_ab, 1) * w * (int64_t)sizeof(u64) > KS_BUDGET) {
		w >>= 1;
	}
	while (w > 64 && searches <= w / 2) {
		w >>= 1;
	}
	return w;
}

int ks_check_call(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const pgq_options *opts, int64_t k,
                  const int64_t *out_npaths, const int64_t *out_first_path, const uint8_t *out_valid,
                  int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (!out_path_offsets || !out_elems || !out_total_paths) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	*out_path_offsets = nullptr;
	*out_elems = nullptr;
	*out_total_paths = 0;
	if (p < 0 || (p > 0 && (!src || !dst))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (p > 0 && (!out_npaths || !out_first_path || !out_valid)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	if (k < 1) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "k must be >= 1");
	}
	if (opts && (opts->lanes < 0 || opts->lanes > 512 || opts->lanes % 64)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "lanes must be 0 or a multiple of 64 up to 512");
	}
	if (p >= 0x7fffffffLL) {
		return pgq_fail(PGQ_ERR_RANGE, "too many pairs in one call");
	}
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	if (opts && opts->shard_count > 1) {
		return pgq_fail(PGQ_ERR_UNSUPPORTED, "shortest_k_paths has no multi-GPU form");
	}
	return PGQ_OK;
}

// What a shortest_k_groups call asks of the walk driver on top of shortest_k_paths' outputs: k counts length groups,
// max_paths cuts the lists, and the per-row group results (host arrays of p; count nullable).  count_only stops after
// the counting pass, with out_valid = the row has a walk.
struct KgCall {
	int64_t max_paths;
	bool count_only;
	int64_t *count, *ngroups, *last_len;
	uint8_t *complete;
};

// shortest_k_paths (kg null) and WALK's shortest_k_groups: the four phases of the top.  The arguments are checked.
static int ks_run(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                  const uint8_t *dst_valid, const pgq_options *opts, int64_t k, const KgCall *kg, int64_t *out_npaths,
                  int64_t *out_first_path, uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
                  int64_t *out_total_paths, pgq_stats *stats) {
	int64_t budget;
	PGQ_TRY(layer_budget(&budget));
	const int64_t n = csr->n, n_ab = csr->n_ab;
	// the lanes: the rows whose ids are both valid, in input order
	std::vector<int32_t> lane_row;
	for (int64_t i = 0; i < p; i++) {
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		if (src[i] < 0 || src[i] >= n || dst[i] < 0 || dst[i] >= n) {
			return pgq_fail(PGQ_ERR_RANGE, "vertex id outside [0, %lld) in row %lld", (long long)n, (long long)i);
		}
		lane_row.push_back((int32_t)i);
	}
	const int64_t S = (int64_t)lane_row.size();
	const int W = ks_lanes(opts, n_ab, S);
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	st.lanes = W;
	st.searches = S;
	if (p == 0) {
		if (!(kg && kg->count_only)) {
			PGQ_TRY(empty_lists(out_path_offsets, out_elems));
		}
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
	const size_t b8 = (size_t)p * sizeof(int64_t);
	Walk w = {};
	w.csr = csr;
	w.ws = ws;
	w.st = &st;
	w.what = "walks";
	w.in_list = csr->in.adj;
	uint8_t *d_valid;
	PGQ_TRY(stage_column(ws, WS_IN_SRC, src, b8, (const void **)&w.src));
	PGQ_TRY(stage_column(ws, WS_IN_DST, dst, b8, (const void **)&w.dst));
	PGQ_TRY(stage_column(ws, WS_KS_LANE_ROW, S ? lane_row.data() : nullptr, (size_t)S * sizeof(int32_t),
	                     (const void **)&w.lane_row));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_VALID, (size_t)p, (void **)&d_valid));
	PGQ_TRY(walk_reserve_lanes(w, S, W));
	PGQ_TRY(walk_reserve_rows(w, p));
	int64_t *lg = nullptr;
	std::vector<u64> h_total; // shortest_k_groups: each lane's walk count N and its groups past h = 0
	std::vector<int64_t> h_lg;
	if (kg) {
		PGQ_TRY(pgq_ws_reserve(ws, WS_KG_GROUPS, (size_t)W * sizeof(int64_t), (void **)&lg));
		h_total.resize((size_t)S);
		h_lg.resize((size_t)S);
	}
	PGQ_CUDA(cudaEventRecord(ws->ev_begin, s));
	PGQ_CUDA(cudaMemsetAsync(w.npaths, 0, b8, s));
	PGQ_CUDA(cudaMemsetAsync(w.elems_row, 0, b8, s));
	PGQ_CUDA(cudaMemsetAsync(w.last, 0xff, b8, s)); // -1: no walk
	PGQ_CUDA(cudaMemsetAsync(w.alive, 0, (size_t)W * sizeof(uint32_t), s));
	if (S > 0) {
		k_ks_lanes<<<grid_size((S + 255) / 256, 4096), 256, 0, s>>>(S, w.lane_row, w.src, w.dst, csr->perm, w.psrc, w.pdst);
		PGQ_CUDA(cudaGetLastError());
		st.kernel_launches++;
	}
	if (!(kg && kg->count_only)) {
		PGQ_TRY(build_step_lists(csr, ws, s, &w.step_key, &w.step_pos, &st.kernel_launches));
	}
	// ---- per batch: backward reach, then the counting pass ----
	for (int64_t b0 = 0; b0 < S; b0 += W) {
		const int cnt = (int)std::min<int64_t>(W, S - b0);
		const int L = (int)std::min<int64_t>(W, (cnt + 63) / 64 * 64);
		const int bwd = L / 64;
		const int64_t bcells = n * bwd;
		const unsigned lane_grid = grid_size((cnt + 255) / 256, 64);
		const int32_t *lrow = w.lane_row + b0, *psrc = w.psrc + b0, *pdst = w.pdst + b0;
		st.batches++;
		PGQ_CUDA(cudaMemsetAsync(w.reach, 0, (size_t)bcells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(w.front, 0, (size_t)bcells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(w.next, 0, (size_t)bcells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(w.act, 0, (size_t)bwd * sizeof(u64), s));
		if (kg) {
			PGQ_CUDA(cudaMemsetAsync(lg, 0, (size_t)cnt * sizeof(int64_t), s));
		}
		k_ks_reach_seed<<<lane_grid, 256, 0, s>>>(cnt, bwd, pdst, w.reach, w.front);
		PGQ_CUDA(cudaGetLastError());
		st.kernel_launches++;
		PGQ_TRY(walk_reach(w, bwd, bcells, AllEdges()));
		auto start = [&]() {
			k_ks_start<<<lane_grid, 256, 0, s>>>(cnt, bwd, k, lrow, psrc, pdst, w.reach, w.total, w.act, w.npaths,
			                                     w.elems_row, w.last, w.ctr);
		};
		auto step = [&](int h, const u64 *cur) {
			if (kg) {
				k_kg_step<<<lane_grid, 256, 0, s>>>(h, cnt, L, n_ab, k, kg->max_paths, lrow, psrc, pdst, cur, w.alive,
				                                    w.total, lg, w.act, w.npaths, w.elems_row, w.last, w.ctr);
			} else {
				k_ks_step<<<lane_grid, 256, 0, s>>>(h, cnt, L, n_ab, k, lrow, pdst, cur, w.alive, w.total, w.act, w.npaths,
				                                    w.elems_row, w.last, w.ctr);
			}
		};
		PGQ_TRY(walk_count(w, L, cnt, bwd, psrc, AllEdges(), start, step, &st.levels,
		                   "a row needs a walk longer than"));
		if (kg) {
			PGQ_CUDA(cudaMemcpyAsync(h_total.data() + b0, w.total, (size_t)cnt * sizeof(u64), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaMemcpyAsync(h_lg.data() + b0, lg, (size_t)cnt * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
			st.d2h_bytes += cnt * (int64_t)(sizeof(u64) + sizeof(int64_t));
		}
	}
	// ---- the rows' walk counts and element counts; their first walk and first element ----
	std::vector<int64_t> h_np((size_t)p), h_el((size_t)p), h_last((size_t)p);
	PGQ_CUDA(cudaMemcpyAsync(h_np.data(), w.npaths, b8, cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaMemcpyAsync(h_el.data(), w.elems_row, b8, cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaMemcpyAsync(h_last.data(), w.last, b8, cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	st.h2d_bytes += 2 * (int64_t)b8 + S * (int64_t)sizeof(int32_t);
	st.d2h_bytes += 3 * (int64_t)b8;
	if (kg) { // the rows' groups: NULL rows have none and are complete
		std::vector<int64_t> h_count((size_t)p, 0);
		for (int64_t i = 0; i < p; i++) {
			kg->ngroups[i] = 0;
			kg->last_len[i] = -1;
		}
		for (int64_t ln = 0; ln < S; ln++) {
			const int64_t row = lane_row[(size_t)ln];
			h_count[(size_t)row] = (int64_t)h_total[(size_t)ln];
			if (h_total[(size_t)ln]) {
				kg->ngroups[row] = h_lg[(size_t)ln] + (src[row] == dst[row] ? 1 : 0);
				kg->last_len[row] = h_last[(size_t)row];
			}
		}
		if (kg->count) {
			memcpy(kg->count, h_count.data(), b8);
		}
		if (kg->count_only) {
			PGQ_TRY(walk_end(g, &st, "walk counts"));
			for (int64_t i = 0; i < p; i++) {
				out_valid[i] = h_count[(size_t)i] > 0;
			}
			if (stats) {
				*stats = st;
			}
			return PGQ_OK;
		}
		for (int64_t i = 0; i < p; i++) {
			if (kg->max_paths == 0 && (u64)h_count[(size_t)i] == AS_MAX) {
				return pgq_fail(PGQ_ERR_UNSUPPORTED, "row %lld has at least INT64_MAX walks: list them with max_paths > 0",
				                (long long)i);
			}
			kg->complete[i] = h_np[(size_t)i] == h_count[(size_t)i];
		}
	}
	PGQ_TRY(walk_offsets(w, 0, p, h_np.data(), h_el.data(), d_valid));
	// ---- the storing pass and the unranking, group by group over the call's lanes ----
	std::vector<WalkLane> listed;
	for (int64_t ln = 0; ln < S; ln++) {
		const int64_t row = lane_row[(size_t)ln];
		if (h_np[(size_t)row] > 0) {
			listed.push_back({(int32_t)ln, row, h_last[(size_t)row]});
		}
	}
	PGQ_TRY(walk_store(w, listed, W, budget, [](const int32_t *) { return AllEdges(); }));
	PGQ_TRY(walk_lists(w, g, p, d_valid, out_first_path, out_valid, out_path_offsets, out_elems, out_total_paths));
	memcpy(out_npaths, h_np.data(), b8);
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_shortest_k_paths(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                    const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                    int64_t k, int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
                                    int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths,
                                    pgq_stats *stats) {
	PGQ_TRY(ks_check_call(csr, p, src, dst, opts, k, out_npaths, out_first_path, out_valid, out_path_offsets, out_elems,
	                      out_total_paths));
	return ks_run(csr, p, src, dst, src_valid, dst_valid, opts, k, nullptr, out_npaths, out_first_path, out_valid,
	              out_path_offsets, out_elems, out_total_paths, stats);
}

// shortest_k_groups' WALK (pgq_kpaths_modes.cu checks the call and sends WALK here)
int kg_walk(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
            const uint8_t *dst_valid, const pgq_options *opts, int64_t k, int64_t max_paths, int64_t *out_count,
            int64_t *out_ngroups, int64_t *out_last_len, uint8_t *out_complete, int64_t *out_npaths,
            int64_t *out_first_path, uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
            int64_t *out_total_paths, pgq_stats *stats) {
	const KgCall kg = {max_paths, false, out_count, out_ngroups, out_last_len, out_complete};
	return ks_run(csr, p, src, dst, src_valid, dst_valid, opts, k, &kg, out_npaths, out_first_path, out_valid,
	              out_path_offsets, out_elems, out_total_paths, stats);
}

extern "C" int pgq_shortest_k_groups_count(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                           const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                           int64_t k, int64_t *out_count, int64_t *out_ngroups, int64_t *out_last_len,
                                           uint8_t *out_valid, pgq_stats *stats) {
	int64_t *no_offsets, *no_elems, no_total;
	PGQ_TRY(ks_check_call(csr, p, src, dst, opts, k, out_count, out_ngroups, out_valid, &no_offsets, &no_elems,
	                      &no_total));
	if (p > 0 && !out_last_len) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	const KgCall kg = {0, true, out_count, out_ngroups, out_last_len, nullptr};
	return ks_run(csr, p, src, dst, src_valid, dst_valid, opts, k, &kg, nullptr, nullptr, out_valid, nullptr, nullptr,
	              nullptr, stats);
}
