// pgq_cheapest.cu -- cheapest_path_length on the device CSR: the batched Bellman-Ford of
// cheapest_path_length.cpp:12-136 (TemplatedBatchBellmanFord: one lane per row, all lanes of an edge
// relaxed together, sweeps until nothing changes).  sm_90a only.
//
// The reference relaxes in place, sequentially, in CSR order, from EVERY vertex, reached or not; the
// distances it ends with are the greatest fixed point of  d[n] = min(d[n], d[v] + w(v,n))  below its start
// values -- for int64 exactly, for double because fl(a + w) is monotone in a -- and do not depend on the
// relaxation order.  The device relaxes in parallel with atomicMin and sweeps only the dirty vertices,
// those whose distance in some lane changed since they were last relaxed, to the same fixed point, bit
// for bit.  "Unreachable" is the reference's own sentinel max/2 (l.15), added to like any other number
// (no guard, as UpdateOneLane l.29-36 has none), so a weight below zero can improve on it: an unreached
// vertex relaxes max/2 + w into its neighbour, which then holds a valid, huge cost (BIGINT: any w < 0;
// DOUBLE: -inf, or w below about -1.5e292).  A batch therefore starts with only its sources dirty when
// every weight is >= 0, and with every vertex dirty when some weight is below zero (pgq_csr::neg_weights,
// found when the CSR is finalized): the first sweep then relaxes from the unreached vertices as the
// reference does, and a row's result does not depend on the other rows of its batch.
// A NaN sum is never better (new_dist < n_dist is false), so an edge of NaN weight never relaxes; without
// that test a NaN with the sign bit set would win every atomicMin.  A negative cycle anywhere in the graph,
// reachable or not, keeps improving for ~2^62 sweeps here as in the reference: there is no cap.
//
// cheapest_path (no reference function: the weighted form of shortestpath's list) runs the same sweeps and then,
// per batch, a BFS over the edges its final distances d make TIGHT for a lane: the edge at out-CSR position e, v -> u,
// with d(v) + w(e) == d(u), the sum in the weight type's arithmetic (k_bf_sweep's int64 addition; a double sum rounded
// to nearest) and the comparison one of values (so -0.0 == 0.0, and a NaN is equal to nothing).  h(u) is u's BFS depth
// from the source over the lane's tight edges (h(s) = 0; the source is never entered again), and the path is
// shortestpath's tie-break on the tight-edge graph: walking back from t, parent(u) is the smallest ORIGINAL vertex id
// v with h(v) = h(u) - 1 and a tight edge v -> u, and the edge is the first tight position of u in v's adjacency.
// One 64-bit atomicMin of (original id << 32 | position in v's adjacency) per tight edge picks exactly that pair.
// When d(s) = 0, the path's weights summed left to right from 0 in the weight type's arithmetic give the row's
// cheapest_path_length cost bit for bit, and the path has the fewest edges among the cheapest.  d(s) != 0 only through
// the sentinel arithmetic of a weight of -inf (or, for BIGINT, below about -max/2) on an edge into s, or a DOUBLE cycle
// through a -inf edge: the path follows the same rule, but its sum is not promised to be the cost.
//
// cheapest_path_count / all_cheapest_paths (SQL/PGQ's ALL CHEAPEST) run the same sweeps and then, per batch, the walk
// engine of shortest_k_paths (pgq_count.cuh, pgq_kshortest.cu's top) over the tight edges of each lane: a BFS back from
// t over the tight in-edges gives B(t) (s outside it: NULL), and the tight walks from s inside B(t) are counted layer
// by layer.  A lane stops after the layer h where the counts are zero on B(t) (exact), where its total saturates, or
// once h >= |B(t)| with counts still alive: such a walk of |B(t)| edges inside B(t) repeats a vertex, so a tight cycle
// lies on an s -> t route and the count is infinite (INT64_MAX); a list of max_paths > 0 walks counts on until it has
// them.  Then the listed walks are stored and unranked as in shortest_k_paths, their offsets continuing batch to batch.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "pgq_bf.cuh"
#include "pgq_count.cuh"
#include "pgq_tile.cuh"

// dists[src][lane] = 0 for the rows of the batch (InitialiseBellmanFord, l.12-27)
template <bool F64>
__global__ void k_bf_sources(int b0, int cnt, int L, const int64_t *__restrict__ src, const uint8_t *__restrict__ src_valid,
                             const int32_t *__restrict__ perm, int64_t n, u64 *dist, uint32_t *dirty, int *err) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l < cnt) {
		const int64_t row = b0 + l;
		if (!src_valid || src_valid[row]) {
			const int64_t s = src[row];
			if (s < 0 || s >= n) {
				*err = 1;
				return;
			}
			const int ps = perm[s];
			dist[(int64_t)ps * L + l] = F64 ? f64_key(0.0) : 0ull;
			atomicOr(&dirty[ps >> 5], 1u << (ps & 31));
		}
	}
}

// result rows of the batch (l.73-101): max/2 -> NULL, NULL source / target -> NULL
template <bool F64>
__global__ void k_bf_results(int b0, int cnt, int L, const int64_t *__restrict__ dst, const uint8_t *__restrict__ src_valid,
                             const uint8_t *__restrict__ dst_valid, const int32_t *__restrict__ perm, int64_t n,
                             const u64 *__restrict__ dist, int64_t *out, uint8_t *out_valid, int *err) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l < cnt) {
		const int64_t row = b0 + l;
		out_valid[row] = 0;
		out[row] = 0;
		if ((src_valid && !src_valid[row]) || (dst_valid && !dst_valid[row])) {
			return;
		}
		const int64_t d = dst[row];
		if (d < 0 || d >= n) {
			*err = 1;
			return;
		}
		const u64 k = dist[(int64_t)perm[d] * L + l];
		if (F64) {
			const double c = key_f64(k);
			if (c != 1.7976931348623157e308 / 2) {
				out[row] = __double_as_longlong(c);
				out_valid[row] = 1;
			}
		} else if ((long long)k != BF_INF_I64) {
			out[row] = (long long)k;
			out_valid[row] = 1;
		}
	}
}

// What a call does with a batch's distances once its sweeps have ended (cheapest_path_length: nothing more)
struct NoTightSearch {
	int operator()(int b0, int cnt, int L, const u64 *dist) const {
		return PGQ_OK;
	}
};

// Runs the batches.  after(b0, cnt, L, dist) is called behind each batch's results, while dist still holds its
// distances.
template <bool F64, class AfterSweeps>
static int run_bf(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                  const uint8_t *d_sv, const uint8_t *d_dv, int64_t *d_out, uint8_t *d_ov, pgq_stats *st,
                  const AfterSweeps &after) {
	cudaStream_t s = ws->stream;
	const int64_t n = csr->n;
	// lanes per batch: as many as a 2 GB distance array allows, at most 256 (the reference's largest batch)
	int L = 256;
	while (L > 32 && (int64_t)L * std::max<int64_t>(n, 1) * 8 > ((int64_t)2 << 30)) {
		L >>= 1;
	}
	L = (int)std::min<int64_t>(L, ((p + 31) / 32) * 32);
	u64 *dist;
	uint32_t *dirty;
	int *flags, *h_flags;
	const size_t dist_elems = (size_t)std::max<int64_t>(n, 1) * L;
	const size_t dirty_bytes = ((size_t)n / 32 + 1) * sizeof(uint32_t);
	PGQ_TRY(pgq_ws_reserve(ws, WS_BF_DIST, dist_elems * sizeof(u64), (void **)&dist));
	PGQ_TRY(pgq_ws_reserve(ws, WS_BF_DIRTY, dirty_bytes, (void **)&dirty));
	PGQ_TRY(pgq_ws_reserve(ws, WS_BF_FLAGS, 256, (void **)&flags)); // [0] changed, [1] range error
	PGQ_TRY(pgq_ws_pinned(ws, 256, (void **)&h_flags));
	PGQ_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(int), s));
	const int sms = csr->ctx->sm_count;
	for (int64_t b0 = 0; b0 < p; b0 += L) {
		const int cnt = (int)std::min<int64_t>(L, p - b0);
		k_bf_init<F64><<<(unsigned)std::min<int64_t>((dist_elems + 255) / 256, (int64_t)sms * 16), 256, 0, s>>>(
		    (int64_t)dist_elems, dist);
		// a weight below zero can improve on max/2: then the first sweep relaxes from every vertex (see the top)
		PGQ_CUDA(cudaMemsetAsync(dirty, csr->neg_weights ? 0xff : 0, dirty_bytes, s));
		k_bf_sources<F64><<<(cnt + 127) / 128, 128, 0, s>>>((int)b0, cnt, L, d_src, d_sv, csr->perm, n, dist, dirty,
		                                                   flags + 1);
		st->batches++;
		st->kernel_launches += 2;
		for (;;) {
			PGQ_CUDA(cudaMemsetAsync(flags, 0, sizeof(int), s));
			k_bf_sweep<F64><<<(unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, (int64_t)sms * 8)), 256, 0, s>>>(
			    n, L, csr->out.off, csr->out.adj, csr->w_bits, dist, dirty, flags);
			PGQ_CUDA(cudaGetLastError());
			PGQ_CUDA(cudaMemcpyAsync(h_flags, flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st->levels++;
			st->kernel_launches++;
			if (h_flags[1]) {
				return pgq_fail(PGQ_ERR_RANGE, "source rowid outside [0,%lld)", (long long)n);
			}
			if (!h_flags[0]) {
				break;
			}
		}
		k_bf_results<F64><<<(cnt + 127) / 128, 128, 0, s>>>((int)b0, cnt, L, d_dst, d_sv, d_dv, csr->perm, n, dist, d_out,
		                                                   d_ov, flags + 1);
		st->kernel_launches++;
		PGQ_TRY(after((int)b0, cnt, L, dist));
	}
	PGQ_CUDA(cudaMemcpyAsync(h_flags, flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	if (h_flags[1]) {
		return pgq_fail(PGQ_ERR_RANGE, "source or destination rowid outside [0,%lld)", (long long)n);
	}
	st->lanes = L;
	return PGQ_OK;
}

extern "C" int pgq_cheapest_path_length(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                        const uint8_t *src_valid, const uint8_t *dst_valid, void *out_cost,
                                        uint8_t *out_valid, pgq_stats *stats) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (p < 0 || (p > 0 && (!src || !dst || !out_cost || !out_valid))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (!csr->finalized || !csr->w_bits || csr->weight_type == 0) {
		// cheapest_path_length_function_data.cpp:22-24
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing cheapest path");
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
	int64_t *d_src, *d_dst, *d_out;
	uint8_t *d_sv, *d_dv, *d_ov;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	PGQ_TRY(stage_column(ws, WS_IN_SRC, src, b8, (const void **)&d_src));
	PGQ_TRY(stage_column(ws, WS_IN_DST, dst, b8, (const void **)&d_dst));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LEN, b8, (void **)&d_out));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_VALID, (size_t)p, (void **)&d_ov));
	PGQ_TRY(stage_column(ws, WS_IN_VALID, src_valid, (size_t)p, (const void **)&d_sv));
	PGQ_TRY(stage_column(ws, WS_IN_DST_VALID, dst_valid, (size_t)p, (const void **)&d_dv));
	st.h2d_bytes = 2 * (int64_t)b8 + (src_valid ? p : 0) + (dst_valid ? p : 0);
	PGQ_TRY((csr->weight_type == 2) ? run_bf<true>(csr, ws, p, d_src, d_dst, d_sv, d_dv, d_out, d_ov, &st, NoTightSearch())
	                                : run_bf<false>(csr, ws, p, d_src, d_dst, d_sv, d_dv, d_out, d_ov, &st, NoTightSearch()));
	cudaMemcpyAsync(out_cost, d_out, b8, cudaMemcpyDeviceToHost, s);
	cudaMemcpyAsync(out_valid, d_ov, (size_t)p, cudaMemcpyDeviceToHost, s);
	st.d2h_bytes = (int64_t)b8 + p;
	cudaError_t e = cudaStreamSynchronize(s);
	if (e != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) {
		return pgq_fail(PGQ_ERR_CUDA, "cheapest_path_length failed: %s", cudaGetErrorString(e));
	}
	g.settled = true;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

// ---- cheapest_path: the BFS over the tight edges of a batch (see the top) --------------------------------------------
#define TIGHT_UNSET 0xFFFFu   // h not set; a level is at most 0xFFFE
#define TIGHT_NO_PARENT (~0ull) // a parent key no tight edge has written yet

// The counters a seed or level kernel publishes for the host: [0] |F| of the frontier it marked, [1] that frontier's
// out-edges, [2] rows whose target it reached, [3] (seed only) rows open: cost valid, s != t.
enum { TC_FRONTIER = 0, TC_EDGES = 1, TC_REACHED = 2, TC_OPEN = 3 };

// h(s) = 0 for every lane with a source, F_0 = the sources, and each lane's target: its internal id while the row is
// open, -2 for [s] (s == t), -1 for NULL (a NULL or outside id, or a NULL cost).  One thread per lane of the batch.
template <bool F64>
__global__ void k_tight_seed(int b0, int cnt, int L, const int64_t *__restrict__ src, const int64_t *__restrict__ dst,
                             const uint8_t *__restrict__ src_valid, const uint8_t *__restrict__ dst_valid,
                             const int32_t *__restrict__ perm, const int32_t *__restrict__ off, int64_t n,
                             const u64 *__restrict__ dist, uint16_t *level, uint32_t *front, int32_t *lane_tgt,
                             unsigned long long *cnt_out) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l >= L) {
		return;
	}
	int tgt = -1;
	if (l < cnt) {
		const int64_t row = b0 + l;
		const int64_t s = src[row], t = dst[row];
		if ((!src_valid || src_valid[row]) && s >= 0 && s < n) { // (an id outside [0, n) fails the call)
			const int ps = perm[s];
			level[(int64_t)ps * L + l] = 0;
			const uint32_t bit = 1u << (ps & 31);
			if (!(atomicOr(&front[ps >> 5], bit) & bit)) {
				atomicAdd(&cnt_out[TC_FRONTIER], 1ull);
				atomicAdd(&cnt_out[TC_EDGES], (unsigned long long)(off[ps + 1] - off[ps]));
			}
			if ((!dst_valid || dst_valid[row]) && t >= 0 && t < n) {
				const int pt = perm[t];
				const u64 k = dist[(int64_t)pt * L + l];
				if (s == t) {
					tgt = -2;
				} else if (F64 ? key_f64(k) != 1.7976931348623157e308 / 2 : (long long)k != BF_INF_I64) {
					tgt = pt;
					atomicAdd(&cnt_out[TC_OPEN], 1ull);
				}
			}
		}
	}
	lane_tgt[l] = tgt;
}

// Expands F_k: a warp per frontier vertex v, 32 lanes at a time (k_bf_sweep's layout).  For each out-edge v -> u tight
// in a lane with h(v) = k, where h(u) is unset or k + 1: h(u) = k + 1 and the parent key of (u, lane) takes the
// minimum of (original id of v << 32 | position of the edge in v's adjacency).  The one thread whose atomicMin finds
// no key yet has put u into F_k+1 for that lane; the first to set u's bit in `next` counts u and its out-degree.
template <bool F64>
__global__ void __launch_bounds__(256) k_tight_level(int k, int64_t n, int L, const int32_t *__restrict__ off,
                                                     const int32_t *__restrict__ adj, const int64_t *__restrict__ w_bits,
                                                     const int32_t *__restrict__ inv, const u64 *__restrict__ dist,
                                                     uint16_t *level, u64 *pkey, const uint32_t *__restrict__ cur,
                                                     uint32_t *next, const int32_t *__restrict__ lane_tgt,
                                                     unsigned long long *cnt_out) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	const uint16_t hk = (uint16_t)k, hk1 = (uint16_t)(k + 1);
	unsigned long long nf = 0, ne = 0;
	unsigned reached = 0;
	for (int64_t v = warp; v < n; v += nwarps) {
		if (!(cur[v >> 5] & (1u << (v & 31)))) {
			continue;
		}
		const int e0 = off[v], e1 = off[v + 1];
		const u64 base = (u64)(uint32_t)inv[v] << 32;
		for (int g = 0; g < L; g += 32) {
			const int l = g + lane;
			const bool act = level[v * L + l] == hk;
			if (!__any_sync(FULL_MASK, act)) {
				continue;
			}
			const u64 dk = dist[v * L + l];
			const int tgt = lane_tgt[l];
			for (int e = e0; e < e1; e++) {
				const int u = adj[e];
				bool fresh = false;
				if (act) {
					const int64_t slot = (int64_t)u * L + l;
					const uint16_t hu = level[slot];
					if (hu == TIGHT_UNSET || hu == hk1) {
						bool tight;
						if (F64) {
							tight = key_f64(dk) + __longlong_as_double(w_bits[e]) == key_f64(dist[slot]);
						} else {
							tight = dk + (u64)w_bits[e] == dist[slot];
						}
						if (tight) {
							if (hu == TIGHT_UNSET) {
								level[slot] = hk1;
							}
							if (atomicMin(&pkey[slot], base | (u64)(e - e0)) == TIGHT_NO_PARENT) {
								fresh = true;
								reached += (u == tgt);
							}
						}
					}
				}
				if (__any_sync(FULL_MASK, fresh) && lane == 0) {
					const uint32_t bit = 1u << (u & 31);
					if (!(atomicOr(&next[u >> 5], bit) & bit)) {
						nf++;
						ne += (unsigned long long)(off[u + 1] - off[u]);
					}
				}
			}
		}
	}
	reached = __reduce_add_sync(FULL_MASK, reached);
	if (lane == 0 && (nf | reached)) {
		atomicAdd(&cnt_out[TC_FRONTIER], nf);
		atomicAdd(&cnt_out[TC_EDGES], ne);
		atomicAdd(&cnt_out[TC_REACHED], (unsigned long long)reached);
	}
}

// list lengths of the batch's rows: 2 h(t) + 1, 1 for [s], 0 for NULL (k_path_offsets turns them into offsets)
__global__ void k_tight_lengths(int b0, int cnt, int L, const int32_t *__restrict__ lane_tgt,
                                const uint16_t *__restrict__ level, int64_t *out_lengths) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l < cnt) {
		const int tgt = lane_tgt[l];
		int64_t len = 0;
		if (tgt == -2) {
			len = 1;
		} else if (tgt >= 0) {
			const uint16_t h = level[(int64_t)tgt * L + l];
			len = h == TIGHT_UNSET ? 0 : 2 * (int64_t)h + 1;
		}
		out_lengths[b0 + l] = len;
	}
}

// One thread per row of the batch: follows the parent keys back from t and writes [s, e1, v1, ..., ek, t] (original
// vertex ids, edge rowids) at the row's offset.
__global__ void k_tight_walk(int b0, int cnt, int L, const int64_t *__restrict__ src, const int64_t *__restrict__ dst,
                             const int32_t *__restrict__ lane_tgt, const u64 *__restrict__ pkey,
                             const int32_t *__restrict__ perm, const int32_t *__restrict__ off,
                             const int64_t *__restrict__ edge_ids, const int64_t *__restrict__ out_offsets,
                             const int64_t *__restrict__ out_lengths, int64_t *elems) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l >= cnt) {
		return;
	}
	const int64_t row = b0 + l;
	const int64_t len = out_lengths[row];
	if (len == 0) {
		return;
	}
	int64_t *out = elems + out_offsets[row];
	if (len == 1) {
		out[0] = src[row];
		return;
	}
	out[len - 1] = dst[row];
	int cur = lane_tgt[l];
	for (int64_t j = (len - 1) / 2; j >= 1; j--) {
		const u64 key = pkey[(int64_t)cur * L + l];
		const int v_orig = (int)(key >> 32);
		const int v = perm[v_orig];
		out[2 * j - 1] = edge_ids[off[v] + (int)(uint32_t)key];
		out[2 * j - 2] = v_orig;
		cur = v;
	}
}

// The tight search of every batch, behind its sweeps (run_bf's AfterSweeps): levels, parent keys and the walk of the
// batch's rows into the element array, whose offsets continue the previous batch's (rows take lanes in input order).
template <bool F64>
struct TightSearch {
	pgq_csr *csr;
	Workspace *ws;
	const int64_t *d_src, *d_dst;
	const uint8_t *d_sv, *d_dv;
	int64_t *d_offsets, *d_lengths;
	uint8_t *d_valid;
	pgq_stats *st;
	int64_t *total; // elements written so far
	int operator()(int b0, int cnt, int L, const u64 *dist) const {
		cudaStream_t s = ws->stream;
		const int64_t n = csr->n;
		const size_t cells = (size_t)std::max<int64_t>(n, 1) * L;
		const size_t words = (size_t)n / 32 + 1;
		uint16_t *level;
		u64 *pkey;
		uint32_t *front;
		int32_t *lane_tgt;
		unsigned long long *cnt_d, *cnt_h;
		int64_t *d_range;
		PGQ_TRY(pgq_ws_reserve(ws, WS_CP_LEVEL, cells * sizeof(uint16_t), (void **)&level));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CP_PKEY, cells * sizeof(u64), (void **)&pkey));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CP_FRONTIER, 2 * words * sizeof(uint32_t), (void **)&front));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CP_LANE_TGT, (size_t)L * sizeof(int32_t), (void **)&lane_tgt));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CP_COUNTERS, 256, (void **)&cnt_d));
		PGQ_TRY(pgq_ws_reserve(ws, WS_PATH_TOTAL, 256, (void **)&d_range));
		PGQ_TRY(pgq_ws_pinned(ws, 256, (void **)&cnt_h));
		PGQ_CUDA(cudaMemsetAsync(level, 0xff, cells * sizeof(uint16_t), s));
		PGQ_CUDA(cudaMemsetAsync(pkey, 0xff, cells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(front, 0, 2 * words * sizeof(uint32_t), s));
		PGQ_CUDA(cudaMemsetAsync(cnt_d, 0, 4 * sizeof(unsigned long long), s));
		k_tight_seed<F64><<<(L + 127) / 128, 128, 0, s>>>(b0, cnt, L, d_src, d_dst, d_sv, d_dv, csr->perm, csr->out.off, n,
		                                                 dist, level, front, lane_tgt, cnt_d);
		st->kernel_launches++;
		PGQ_CUDA(cudaMemcpyAsync(cnt_h, cnt_d, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		unsigned long long nf = cnt_h[TC_FRONTIER], ne = cnt_h[TC_EDGES], open = cnt_h[TC_OPEN];
		const int sms = csr->ctx->sm_count;
		uint32_t *cur = front, *next = front + words;
		// F_k is expanded while it holds a vertex and some row is still open; h is uint16 with 0xFFFF for "unset"
		for (int k = 0; nf > 0 && open > 0; k++) {
			if (k >= 0xFFFE) {
				return pgq_fail(PGQ_ERR_UNSUPPORTED, "cheapest path deeper than 65534 edges is not supported");
			}
			st->push_levels++;
			st->frontier_vertices += (int64_t)nf;
			st->edges_traversed += (int64_t)ne;
			PGQ_CUDA(cudaMemsetAsync(next, 0, words * sizeof(uint32_t), s));
			PGQ_CUDA(cudaMemsetAsync(cnt_d, 0, 3 * sizeof(unsigned long long), s));
			k_tight_level<F64><<<(unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, (int64_t)sms * 8)), 256, 0, s>>>(
			    k, n, L, csr->out.off, csr->out.adj, csr->w_bits, csr->inv, dist, level, pkey, cur, next, lane_tgt, cnt_d);
			PGQ_CUDA(cudaGetLastError());
			PGQ_CUDA(cudaMemcpyAsync(cnt_h, cnt_d, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st->kernel_launches++;
			nf = cnt_h[TC_FRONTIER];
			ne = cnt_h[TC_EDGES];
			open -= cnt_h[TC_REACHED];
			std::swap(cur, next);
		}
		k_tight_lengths<<<(cnt + 127) / 128, 128, 0, s>>>(b0, cnt, L, lane_tgt, level, d_lengths);
		pgq_path_offsets(*total, b0, (int64_t)b0 + cnt, d_offsets, d_lengths, d_valid, d_range, s);
		int64_t range = 0;
		PGQ_CUDA(cudaMemcpyAsync(&range, d_range, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		int64_t *elems;
		PGQ_TRY(pgq_ws_grow(ws, WS_ELEMS, (size_t)(*total + range) * sizeof(int64_t), (size_t)*total * sizeof(int64_t), s,
		                    (void **)&elems));
		k_tight_walk<<<(cnt + 127) / 128, 128, 0, s>>>(b0, cnt, L, d_src, d_dst, lane_tgt, pkey, csr->perm, csr->out.off,
		                                              csr->edge_ids, d_offsets, d_lengths, elems);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches += 3;
		*total += range;
		return PGQ_OK;
	}
};

extern "C" int pgq_cheapest_path(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                 const uint8_t *src_valid, const uint8_t *dst_valid, int64_t *out_offsets,
                                 int64_t *out_lengths, uint8_t *out_valid, int64_t **out_elems, int64_t *out_total,
                                 pgq_stats *stats) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (p < 0 || !out_elems || !out_total || (p > 0 && (!src || !dst || !out_offsets || !out_lengths || !out_valid))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	*out_elems = nullptr;
	*out_total = 0;
	if (!csr->finalized || !csr->w_bits || csr->weight_type == 0) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing cheapest path");
	}
	if (p >= 0x7fffffffLL) {
		return pgq_fail(PGQ_ERR_RANGE, "too many pairs in one call");
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
	int64_t *d_src, *d_dst, *d_cost, *d_off, *d_lens;
	uint8_t *d_sv, *d_dv, *d_cv, *d_ov;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	PGQ_TRY(stage_column(ws, WS_IN_SRC, src, b8, (const void **)&d_src));
	PGQ_TRY(stage_column(ws, WS_IN_DST, dst, b8, (const void **)&d_dst));
	PGQ_TRY(stage_column(ws, WS_IN_VALID, src_valid, (size_t)p, (const void **)&d_sv));
	PGQ_TRY(stage_column(ws, WS_IN_DST_VALID, dst_valid, (size_t)p, (const void **)&d_dv));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LEN, b8, (void **)&d_cost)); // the costs, which the sweeps write as for the lengths
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_VALID, (size_t)p, (void **)&d_cv));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_PATH_OFFSETS, b8, (void **)&d_off));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LENGTHS, b8, (void **)&d_lens));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_PATH_VALID, (size_t)p, (void **)&d_ov));
	st.h2d_bytes = 2 * (int64_t)b8 + (src_valid ? p : 0) + (dst_valid ? p : 0);
	int64_t total = 0;
	if (csr->weight_type == 2) {
		const TightSearch<true> tight {csr, ws, d_src, d_dst, d_sv, d_dv, d_off, d_lens, d_ov, &st, &total};
		PGQ_TRY(run_bf<true>(csr, ws, p, d_src, d_dst, d_sv, d_dv, d_cost, d_cv, &st, tight));
	} else {
		const TightSearch<false> tight {csr, ws, d_src, d_dst, d_sv, d_dv, d_off, d_lens, d_ov, &st, &total};
		PGQ_TRY(run_bf<false>(csr, ws, p, d_src, d_dst, d_sv, d_dv, d_cost, d_cv, &st, tight));
	}
	int64_t *h_elems = (int64_t *)malloc((size_t)(total > 0 ? total : 1) * sizeof(int64_t));
	if (!h_elems) {
		return pgq_fail(PGQ_ERR_OOM, "host allocation of %lld path elements failed", (long long)total);
	}
	cudaError_t e = cudaSuccess;
	if (total > 0) {
		e = cudaMemcpyAsync(h_elems, ws->buf[WS_ELEMS], (size_t)total * sizeof(int64_t), cudaMemcpyDeviceToHost, s);
	}
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_offsets, d_off, b8, cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_lengths, d_lens, b8, cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_valid, d_ov, (size_t)p, cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	g.settled = (e == cudaSuccess);
	if (e != cudaSuccess) {
		cudaGetLastError();
		free(h_elems);
		return pgq_fail(PGQ_ERR_CUDA, "copying cheapest paths back failed: %s", cudaGetErrorString(e));
	}
	st.d2h_bytes = 2 * (int64_t)b8 + p + total * (int64_t)sizeof(int64_t);
	*out_elems = h_elems;
	*out_total = total;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

// ---- cheapest_path_count / all_cheapest_paths: the walk engine over the tight edges of a batch (see the top) ---------
// The tight edges of a batch as the walk kernels' edge filter (pgq_count.cuh).  The kernels walk the step lists, whose
// entry e carries the out-CSR position pos[e] of its edge, and so its weight; kernel lane l is lane lane_map[l] of the
// batch (l itself without a map).  The rule is k_tight_level's: d(from) + w == d(to) in the weight type's arithmetic.
template <bool F64>
struct TightEdges {
	const u64 *dist;
	int L;
	const int64_t *w_bits;
	const int32_t *pos;
	const int32_t *lane_map;
	__device__ __forceinline__ bool edge(int64_t e, int64_t from, int64_t to, int l) const {
		const int bl = lane_map ? lane_map[l] : l;
		const u64 dv = dist[from * L + bl], du = dist[to * L + bl];
		const int64_t w = w_bits[pos[e]];
		if (F64) {
			return key_f64(dv) + __longlong_as_double(w) == key_f64(du);
		}
		return dv + (u64)w == du;
	}
	__device__ __forceinline__ u64 lanes(int64_t e, int64_t from, int64_t to, int j, u64 cand) const {
		u64 out = 0;
		while (cand) {
			const int b = __ffsll((long long)cand) - 1;
			cand &= cand - 1;
			if (edge(e, from, to, j * 64 + b)) {
				out |= 1ull << b;
			}
		}
		return out;
	}
};

// par[e] = the internal id of the parent of step-list entry e: the in-lists the tight kernels walk in place of in_adj,
// so that entry e's out-CSR position is step_pos[e].  A warp per in-list.
__global__ void __launch_bounds__(256) k_ac_step_par(int64_t n, int64_t n_ab, const int32_t *__restrict__ in_off,
                                                     const u64 *__restrict__ step_key, const int32_t *__restrict__ perm,
                                                     int32_t *par) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < n_ab; u += nwarps) {
		const u64 key0 = (u64)u * (u64)n;
		for (int e = in_off[u] + lane; e < in_off[u + 1]; e += 32) {
			par[e] = perm[(int)(step_key[e] - key0)];
		}
	}
}

// Each lane of the batch: its row, its internal ids, and whether it is open -- both ids valid and s == t or a cost at t
// (k_tight_seed's rule).  An open lane seeds its target into the backward reach.  One thread per lane.
template <bool F64>
__global__ void k_ac_lanes(int b0, int cnt, int L, int wd, const int64_t *__restrict__ src, const int64_t *__restrict__ dst,
                           const uint8_t *__restrict__ src_valid, const uint8_t *__restrict__ dst_valid,
                           const int32_t *__restrict__ perm, int64_t n, const u64 *__restrict__ dist, int32_t *psrc,
                           int32_t *pdst, int32_t *lane_row, uint32_t *open, u64 *reach, u64 *front) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l >= cnt) {
		return;
	}
	const int64_t row = b0 + l;
	const int64_t s = src[row], t = dst[row];
	int ps = 0, pt = 0;
	bool op = false;
	if ((!src_valid || src_valid[row]) && (!dst_valid || dst_valid[row]) && s >= 0 && s < n && t >= 0 && t < n) {
		ps = perm[s];
		pt = perm[t];
		const u64 k = dist[(int64_t)pt * L + l];
		op = s == t || (F64 ? key_f64(k) != 1.7976931348623157e308 / 2 : (long long)k != BF_INF_I64);
	}
	lane_row[l] = (int32_t)row;
	psrc[l] = ps;
	pdst[l] = pt;
	open[l] = op;
	if (op) {
		const int64_t cell = (int64_t)pt * wd + (l >> 6);
		atomicOr(&reach[cell], 1ull << (l & 63));
		atomicOr(&front[cell], 1ull << (l & 63));
	}
}

// |B_tight(t)| of each lane: a thread per lane, a block per slice of the vertices
__global__ void k_ac_bsize(int64_t n, int wd, const u64 *__restrict__ reach, unsigned long long *bsize) {
	const int l = threadIdx.x;
	unsigned long long c = 0;
	for (int64_t v = blockIdx.x; v < n; v += gridDim.x) {
		c += (reach[v * wd + (l >> 6)] >> (l & 63)) & 1;
	}
	if (c) {
		atomicAdd(&bsize[l], c);
	}
}

// Layer 0 of each lane: NULL unless the lane is open and s lies in B_tight(t); then the lane counts, with [s] as its walk
// of 0 edges when s == t
__global__ void k_ac_start(int cnt, int wd, bool list, const int32_t *__restrict__ lane_row,
                           const int32_t *__restrict__ psrc, const int32_t *__restrict__ pdst,
                           const uint32_t *__restrict__ open, const u64 *__restrict__ reach, u64 *total, uint32_t *inf,
                           u64 *act, int64_t *count, int64_t *npaths, int64_t *elems, int64_t *last, u64 *ctr) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		const int row = lane_row[l];
		const int s = psrc[l], t = pdst[l];
		const bool in_b = open[l] && ((reach[(int64_t)s * wd + (l >> 6)] >> (l & 63)) & 1);
		const int64_t c0 = in_b && s == t ? 1 : 0;
		total[l] = c0;
		inf[l] = 0;
		count[row] = c0;
		npaths[row] = list ? c0 : 0;
		elems[row] = list ? c0 : 0;
		last[row] = c0 ? 0 : -1;
		if (in_b) {
			atomicOr(&act[l >> 6], 1ull << (l & 63));
			atomicAdd(&ctr[KS_ACTIVE], 1ull);
		}
	}
}

// After layer h: each counting lane adds its count c at t to its saturating total and lists min(c, the room under
// max_paths) walks of h edges (all c for max_paths = 0; none for a count).  It stops after the layer where w_h was zero
// on B_tight(t) (the count is exact), where its total saturates, or once w_h is alive at h >= |B_tight(t)| (the count is
// infinite: DESIGN.md section 3) -- at once when it lists nothing more or max_paths = 0, else when it has max_paths walks.
__global__ void k_ac_step(int h, int cnt, int L, int64_t n_ab, bool list, int64_t max_paths,
                          const int32_t *__restrict__ lane_row, const int32_t *__restrict__ pdst,
                          const u64 *__restrict__ cur, const unsigned long long *__restrict__ bsize, uint32_t *alive,
                          u64 *total, uint32_t *inf, u64 *act, int64_t *count, int64_t *npaths, int64_t *elems,
                          int64_t *last, u64 *ctr) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		if (!((act[l >> 6] >> (l & 63)) & 1)) {
			continue;
		}
		const int row = lane_row[l];
		const int t = pdst[l];
		const u64 c = t < n_ab ? cur[(int64_t)t * L + l] : 0;
		const u64 tot = sat_add(total[l], c);
		total[l] = tot;
		const u64 listed = (u64)npaths[row];
		const u64 take = !list ? 0 : max_paths ? min(c, (u64)max_paths - listed) : c;
		if (take) {
			npaths[row] = (int64_t)sat_add(listed, take);
			elems[row] = (int64_t)sat_add((u64)elems[row], sat_mul_len(take, 2 * (int64_t)h + 1));
			last[row] = h;
		}
		const bool live = alive[l] != 0;
		alive[l] = 0;
		const bool infinite = inf[l] || (live && (u64)h >= (u64)bsize[l]);
		inf[l] = infinite;
		count[row] = infinite ? (int64_t)AS_MAX : (int64_t)tot;
		const bool stop = !live || tot == AS_MAX || (infinite && (!list || max_paths == 0 || listed + take >= (u64)max_paths));
		if (h >= KS_WALK_MAX && !stop) {
			ctr[KS_TOO_LONG] = 1;
		}
		if (stop) {
			atomicAnd(&act[l >> 6], ~(1ull << (l & 63)));
		} else {
			atomicAdd(&ctr[KS_ACTIVE], 1ull);
		}
	}
}

// What both calls keep across the batches: the walk engine, the per-row counts on the device ([p]) and the call's choices
struct AcCall {
	Walk w;
	bool list;
	int64_t max_paths, budget;
	int64_t *count;
	uint8_t *valid;
};

// The tight walk search of every batch, behind its sweeps (run_bf's AfterSweeps): the tight backward reach, the counting
// pass, and for the lists the storing pass and the unranking, whose offsets continue the previous batch's.
template <bool F64>
struct TightWalks {
	const uint8_t *d_sv, *d_dv;
	AcCall *call;
	int operator()(int b0, int cnt, int L, const u64 *dist) const {
		Walk &w = call->w;
		pgq_csr *csr = w.csr;
		Workspace *ws = w.ws;
		cudaStream_t s = ws->stream;
		const int64_t n = csr->n, n_ab = csr->n_ab;
		const int wd = (L + 63) / 64;
		const int64_t cells = std::max<int64_t>(n, 1) * wd;
		int32_t *lane_row;
		uint32_t *open, *inf;
		unsigned long long *bsize;
		PGQ_TRY(walk_reserve_lanes(w, L, L));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KS_LANE_ROW, (size_t)L * sizeof(int32_t), (void **)&lane_row));
		PGQ_TRY(pgq_ws_reserve(ws, WS_AC_OPEN, (size_t)L * sizeof(uint32_t), (void **)&open));
		PGQ_TRY(pgq_ws_reserve(ws, WS_AC_BSIZE, (size_t)L * sizeof(u64), (void **)&bsize));
		PGQ_TRY(pgq_ws_reserve(ws, WS_AC_INF, (size_t)L * sizeof(uint32_t), (void **)&inf));
		w.lane_row = lane_row;
		PGQ_CUDA(cudaMemsetAsync(w.reach, 0, (size_t)cells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(w.front, 0, (size_t)cells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(w.next, 0, (size_t)cells * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(bsize, 0, (size_t)L * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(w.alive, 0, (size_t)L * sizeof(uint32_t), s));
		PGQ_CUDA(cudaMemsetAsync(w.act, 0, (size_t)wd * sizeof(u64), s));
		const TightEdges<F64> tight {dist, L, csr->w_bits, w.step_pos, nullptr};
		k_ac_lanes<F64><<<(cnt + 127) / 128, 128, 0, s>>>(b0, cnt, L, wd, w.src, w.dst, d_sv, d_dv, csr->perm, n, dist, w.psrc,
		                                                 w.pdst, lane_row, open, w.reach, w.front);
		PGQ_CUDA(cudaGetLastError());
		w.st->kernel_launches++;
		PGQ_TRY(walk_reach(w, wd, cells, tight));
		k_ac_bsize<<<grid_size(n, (int64_t)csr->ctx->sm_count * 8), L, 0, s>>>(n, wd, w.reach, bsize);
		w.st->kernel_launches++;
		auto start = [&]() {
			k_ac_start<<<(cnt + 255) / 256, 256, 0, s>>>(cnt, wd, call->list, lane_row, w.psrc, w.pdst, open, w.reach, w.total,
			                                             inf, w.act, call->count, w.npaths, w.elems_row, w.last, w.ctr);
		};
		auto step = [&](int h, const u64 *cur) {
			k_ac_step<<<(cnt + 255) / 256, 256, 0, s>>>(h, cnt, L, n_ab, call->list, call->max_paths, lane_row, w.pdst, cur,
			                                            bsize, w.alive, w.total, inf, w.act, call->count, w.npaths,
			                                            w.elems_row, w.last, w.ctr);
		};
		PGQ_TRY(walk_count(w, L, cnt, wd, w.psrc, tight, start, step, &w.st->pull_levels,
		                   "a row still counts cheapest paths after"));
		if (!call->list) {
			return PGQ_OK;
		}
		// ---- the batch's walks and elements: checked, then placed behind the previous batches' ----
		std::vector<int64_t> h_count((size_t)cnt), h_np((size_t)cnt), h_el((size_t)cnt), h_last((size_t)cnt);
		PGQ_CUDA(cudaMemcpyAsync(h_count.data(), call->count + b0, (size_t)cnt * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaMemcpyAsync(h_np.data(), w.npaths + b0, (size_t)cnt * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaMemcpyAsync(h_el.data(), w.elems_row + b0, (size_t)cnt * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaMemcpyAsync(h_last.data(), w.last + b0, (size_t)cnt * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		w.st->d2h_bytes += 4 * cnt * (int64_t)sizeof(int64_t);
		for (int l = 0; l < cnt; l++) {
			if (call->max_paths == 0 && (u64)h_count[(size_t)l] == AS_MAX) {
				return pgq_fail(PGQ_ERR_UNSUPPORTED, "row %lld has INT64_MAX or infinitely many cheapest paths: list them with "
				                "max_paths > 0", (long long)(b0 + l));
			}
		}
		PGQ_TRY(walk_offsets(w, b0, (int64_t)b0 + cnt, h_np.data(), h_el.data(), call->valid));
		// ---- the storing pass and the unranking, group by group over the batch's lanes ----
		std::vector<WalkLane> listed;
		for (int l = 0; l < cnt; l++) {
			if (h_np[(size_t)l] > 0) {
				listed.push_back({l, (int64_t)b0 + l, h_last[(size_t)l]});
			}
		}
		return walk_store(w, listed, L, call->budget, [&](const int32_t *glane) {
			return TightEdges<F64> {dist, L, csr->w_bits, w.step_pos, glane};
		});
	}
};

// Both calls: the arguments are checked; list = false is cheapest_path_count (the list outputs unused)
static int ac_run(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                  const uint8_t *dst_valid, bool list, int64_t max_paths, int64_t *out_count, int64_t *out_npaths,
                  int64_t *out_first_path, uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
                  int64_t *out_total_paths, pgq_stats *stats) {
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	if (p == 0) {
		if (list) {
			PGQ_TRY(empty_lists(out_path_offsets, out_elems));
		}
		if (stats) {
			*stats = st;
		}
		return PGQ_OK;
	}
	AcCall call = {};
	call.list = list;
	call.max_paths = max_paths;
	PGQ_TRY(layer_budget(&call.budget));
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	const int64_t n = csr->n, n_ab = csr->n_ab;
	Walk &w = call.w;
	w.csr = csr;
	w.ws = ws;
	w.st = &st;
	w.what = "cheapest paths";
	int64_t *d_cost;
	uint8_t *d_sv, *d_dv, *d_cv;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	PGQ_CUDA(cudaEventRecord(ws->ev_begin, s));
	PGQ_TRY(stage_column(ws, WS_IN_SRC, src, b8, (const void **)&w.src));
	PGQ_TRY(stage_column(ws, WS_IN_DST, dst, b8, (const void **)&w.dst));
	PGQ_TRY(stage_column(ws, WS_IN_VALID, src_valid, (size_t)p, (const void **)&d_sv));
	PGQ_TRY(stage_column(ws, WS_IN_DST_VALID, dst_valid, (size_t)p, (const void **)&d_dv));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LEN, b8, (void **)&d_cost)); // the sweeps' costs
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_VALID, (size_t)p, (void **)&d_cv));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_PATH_VALID, (size_t)p, (void **)&call.valid));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AC_COUNT, b8, (void **)&call.count));
	PGQ_TRY(walk_reserve_rows(w, p));
	st.h2d_bytes = 2 * (int64_t)b8 + (src_valid ? p : 0) + (dst_valid ? p : 0);
	// the step lists, and each entry's parent: the tight kernels' in-lists
	int32_t *step_par;
	PGQ_TRY(build_step_lists(csr, ws, s, &w.step_key, &w.step_pos, &st.kernel_launches));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AC_STEP_PAR, (size_t)std::max<int64_t>(csr->m, 1) * sizeof(int32_t), (void **)&step_par));
	if (csr->m > 0) {
		k_ac_step_par<<<grid_size((n_ab + 7) / 8, (int64_t)csr->ctx->sm_count * 16), 256, 0, s>>>(n, n_ab, csr->in.off,
		                                                                                       w.step_key, csr->perm,
		                                                                                       step_par);
		PGQ_CUDA(cudaGetLastError());
		st.kernel_launches++;
	}
	w.in_list = step_par;
	if (csr->weight_type == 2) {
		PGQ_TRY(run_bf<true>(csr, ws, p, w.src, w.dst, d_sv, d_dv, d_cost, d_cv, &st, TightWalks<true> {d_sv, d_dv, &call}));
	} else {
		PGQ_TRY(run_bf<false>(csr, ws, p, w.src, w.dst, d_sv, d_dv, d_cost, d_cv, &st, TightWalks<false> {d_sv, d_dv, &call}));
	}
	PGQ_CUDA(cudaMemcpyAsync(out_count, call.count, b8, cudaMemcpyDeviceToHost, s));
	if (!list) {
		PGQ_TRY(walk_end(g, &st, "cheapest path counts"));
		for (int64_t i = 0; i < p; i++) {
			out_valid[i] = out_count[i] > 0;
		}
		st.d2h_bytes += (int64_t)b8 + p;
		if (stats) {
			*stats = st;
		}
		return PGQ_OK;
	}
	PGQ_CUDA(cudaMemcpyAsync(out_npaths, w.npaths, b8, cudaMemcpyDeviceToHost, s));
	st.d2h_bytes += 3 * (int64_t)b8; // the counts, walks and first walks (walk_lists counts the rest)
	PGQ_TRY(walk_lists(w, g, p, call.valid, out_first_path, out_valid, out_path_offsets, out_elems, out_total_paths));
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

// pgq_cheapest_path's argument checks, and max_paths
static int ac_check_call(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, int64_t max_paths,
                         const int64_t *out_count, const uint8_t *out_valid) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (p < 0 || (p > 0 && (!src || !dst || !out_count || !out_valid))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (max_paths < 0) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "max_paths must be >= 0");
	}
	if (!csr->finalized || !csr->w_bits || csr->weight_type == 0) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing cheapest path");
	}
	if (p >= 0x7fffffffLL) {
		return pgq_fail(PGQ_ERR_RANGE, "too many pairs in one call");
	}
	return PGQ_OK;
}

extern "C" int pgq_cheapest_path_count(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                       const uint8_t *src_valid, const uint8_t *dst_valid, int64_t *out_count,
                                       uint8_t *out_valid, pgq_stats *stats) {
	PGQ_TRY(ac_check_call(csr, p, src, dst, 0, out_count, out_valid));
	return ac_run(csr, p, src, dst, src_valid, dst_valid, false, 0, out_count, nullptr, nullptr, out_valid, nullptr,
	              nullptr, nullptr, stats);
}

extern "C" int pgq_all_cheapest_paths(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                      const uint8_t *src_valid, const uint8_t *dst_valid, int64_t max_paths,
                                      int64_t *out_count, int64_t *out_npaths, int64_t *out_first_path,
                                      uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
                                      int64_t *out_total_paths, pgq_stats *stats) {
	if (!out_path_offsets || !out_elems || !out_total_paths) {
		return pgq_fail(csr ? PGQ_ERR_INVALID_ARG : PGQ_ERR_INVALID_ID, "null output");
	}
	*out_path_offsets = nullptr;
	*out_elems = nullptr;
	*out_total_paths = 0;
	PGQ_TRY(ac_check_call(csr, p, src, dst, max_paths, out_count, out_valid));
	if (p > 0 && (!out_npaths || !out_first_path)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	return ac_run(csr, p, src, dst, src_valid, dst_valid, true, max_paths, out_count, out_npaths, out_first_path,
	              out_valid, out_path_offsets, out_elems, out_total_paths, stats);
}
