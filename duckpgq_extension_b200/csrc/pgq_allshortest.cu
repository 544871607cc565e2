// pgq_allshortest.cu -- shortest_path_count and all_shortest_paths on the device CSR: every shortest path of a row
// (SQL/PGQ's ALL SHORTEST, which the reference rejects).  No reference function.  sm_90a only.
//
// The call runs shortestpath's BFS unchanged (pgq_bfs.cu: lane assignment, batches, level loop, path mode) and, per
// batch, while the batch's level array level[v][l] is live, a PathHook in place of shortestpath's walk:
//   * sigma.  sigma(u, l) = the number of shortest paths from the lane's source to u = the sum of sigma(v, l) over the
//     in-edges v -> u (one term per edge, so parallel edges count apart) with level(v, l) = level(u, l) - 1, and
//     sigma(src, l) = 1.  k_sigma_level computes level k = 1 .. K of every lane of the batch, one launch per level, as a
//     deterministic pull over the in-CSC: a warp per vertex u, 32 lanes at a time.  level is vertex-major ([v * L + l]),
//     so a warp reads u's levels and, per in-edge, the parent's levels and counts as 64 B and 256 B runs; a push over
//     the frontier would have to scatter its sums into the same rows with a 64-bit CAS loop per (edge, lane).  Sums
//     saturate at INT64_MAX (the operands are non-negative, so saturating addition is associative and the pull's order
//     does not matter).  Only the lane's source has level 0, so sigma is not stored for level 0: it reads as 1.  A vertex
//     at a level >= 1 has an in-edge, so its internal id lies below n_ab and sigma has n_ab rows.
//   * premise: when a batch stops, every vertex at a level <= K of lane l has its level recorded, and no vertex has a
//     level below its BFS depth.  A batch stops only behind a complete level, and K (the largest target level of the
//     batch's answered rows) is at most the levels it ran.  Every bit that becomes new in a level records the level:
//     k_update_sparse, k_tail (each of its levels is whole) and the bottom-up levels (record_levels /
//     record_levels_warp) all store it.  A bottom-up level skips only finished vertex rows, whose every live lane is
//     seen already, so it skips no new bit.  The one wrong store, a source re-entered through a cycle, is put back to 0
//     by k_path_fix_sources before the hook runs.
//   * counts.  count(row) = sigma(t, lane) (1 for s == t), read by k_as_rows for the rows on the batch's lanes; rows
//     share lanes through source de-duplication.
//   * lists (all_shortest_paths).  k_as_rows also gives each row its number of lists min(count, max_paths) (all of them
//     for max_paths = 0), its element count and a slot in shortestpath's walk buffer; the host brings back the call's
//     running element total (one sync per batch), grows the buffer and k_as_unrank writes the lists.  A warp per
//     (row, rank r) walks back from t: at node u, level k, it scans u's in-edges in step order -- the parent's ORIGINAL
//     id, then the edge's position in the parent's adjacency -- and takes the first edge whose parent v has level k - 1
//     and r < sigma(v), subtracting the sigma of every such edge it passes; a warp scans 32 edges per step with a
//     saturating prefix sum, so a step costs O(in-degree / 32).  Path 0 is shortestpath's path.  Ranks stay exact under
//     saturation: every rank asked for is below INT64_MAX (max_paths = 0 fails on a saturated count); a prefix sum
//     passes r only when its exact value does, because a saturated sum is INT64_MAX > r; and whatever is subtracted is a
//     prefix at most r, which holds no saturated term.  The step order needs in-lists sorted by (original parent id,
//     out position), while the in-CSC is sorted by internal id: the call sorts the out-edges once into step lists with
//     radix_sort_pairs before its BFS starts.  Behind the last batch shortestpath's k_path_offsets / k_path_trivial /
//     k_path_place place every row's lists in row order.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "pgq_count.cuh"
#include "pgq_tile.cuh"

#define AS_UNSET 0xFFFFu // level of a vertex the lane has not reached

// The batch counters a hook brings back: [0] K, the largest target level of the batch's rows; [1] the call's running
// element total (saturating); [2] a row with max_paths = 0 saturated its count.
enum { AS_K = 0, AS_TOTAL = 1, AS_SATURATED = 2 };

// count = lists = list length = 1 for the rows with a valid source and s == t, 0 for the others (the rows on a lane
// are overwritten by their batch)
__global__ void k_as_init_rows(int64_t p, const int64_t *__restrict__ src, const int64_t *__restrict__ dst,
                               const uint8_t *__restrict__ valid, int64_t *count, int64_t *npaths, int64_t *plen) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p; i += (int64_t)gridDim.x * blockDim.x) {
		const int64_t one = ((!valid || valid[i]) && src[i] == dst[i]) ? 1 : 0;
		count[i] = one;
		npaths[i] = one;
		plen[i] = one;
	}
}

// K: the largest level of a target among the batch's rows
__global__ void k_as_depth(int b0, int L, const int32_t *__restrict__ batch_rows, const int *__restrict__ batch_n,
                           const int32_t *__restrict__ row_lane, const int32_t *__restrict__ pdst,
                           const uint16_t *__restrict__ level, u64 *ctr) {
	const int nb = *batch_n;
	unsigned k = 0;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nb; j += gridDim.x * blockDim.x) {
		const int row = batch_rows[j];
		const uint16_t lv = level[(int64_t)pdst[row] * L + (row_lane[row] - b0)];
		k = lv == AS_UNSET ? k : max(k, (unsigned)lv);
	}
	k = __reduce_max_sync(FULL_MASK, k);
	if ((threadIdx.x & 31) == 0 && k) {
		atomicMax(&ctr[AS_K], (u64)k);
	}
}

// Level k of sigma: a warp per vertex u with in-edges, 32 lanes at a time (see the top)
__global__ void __launch_bounds__(256) k_sigma_level(int k, int64_t n_ab, int L, const int32_t *__restrict__ in_off,
                                                     const int32_t *__restrict__ in_adj,
                                                     const uint16_t *__restrict__ level, int64_t *sigma) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	const uint16_t hk = (uint16_t)k, hp = (uint16_t)(k - 1);
	for (int64_t u = warp; u < n_ab; u += nwarps) {
		const int e0 = in_off[u], e1 = in_off[u + 1];
		for (int g = 0; g < L; g += 32) {
			const int l = g + lane;
			const bool act = level[u * L + l] == hk;
			if (!__any_sync(FULL_MASK, act)) {
				continue;
			}
			u64 sum = 0;
			for (int e = e0; e < e1; e++) {
				const int64_t cell = (int64_t)in_adj[e] * L + l;
				if (act && level[cell] == hp) {
					sum = sat_add(sum, k == 1 ? 1ull : (u64)sigma[cell]);
				}
			}
			if (act) {
				sigma[u * L + l] = (int64_t)sum;
			}
		}
	}
}

// The rows of the batch: count, lists, list length; with `lists` also each row's element count (out_lengths, as
// shortestpath's: 1 = [src], written by k_path_trivial) and its slot in the walk buffer
__global__ void k_as_rows(int b0, int L, const int32_t *__restrict__ batch_rows, const int *__restrict__ batch_n,
                          const int32_t *__restrict__ row_lane, const int32_t *__restrict__ psrc,
                          const int32_t *__restrict__ pdst, const uint16_t *__restrict__ level,
                          const int64_t *__restrict__ sigma, int64_t max_paths, int lists, int64_t *count,
                          int64_t *npaths, int64_t *plen, int64_t *out_lengths, int64_t *slot_off, u64 *ctr) {
	const int nb = *batch_n;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nb; j += gridDim.x * blockDim.x) {
		const int row = batch_rows[j];
		const int l = row_lane[row] - b0;
		const int t = pdst[row];
		int64_t c = 0, h = -1;
		if (psrc[row] == t) {
			c = 1;
			h = 0;
		} else {
			const uint16_t lv = level[(int64_t)t * L + l];
			if (lv != AS_UNSET) { // (lv >= 1: only the source has level 0)
				h = lv;
				c = sigma[(int64_t)t * L + l];
			}
		}
		const int64_t np = h < 0 ? 0 : (max_paths > 0 ? min(c, max_paths) : c);
		const int64_t len = h < 0 ? 0 : 2 * h + 1;
		count[row] = c;
		npaths[row] = np;
		plen[row] = len;
		if (lists) {
			if (max_paths == 0 && (u64)c == AS_MAX) {
				ctr[AS_SATURATED] = 1;
			}
			const int64_t elems = len == 0 ? 0 : ((u64)np > AS_MAX / (u64)len ? (int64_t)AS_MAX : np * len);
			out_lengths[row] = elems;
			slot_off[row] = elems > 1 ? (int64_t)atomic_sat_add(&ctr[AS_TOTAL], (u64)elems) : 0;
		}
	}
}

// The step lists: every out-edge v -> u at out-CSR position e, keyed u * n + (original id of v), with e as value; a
// stable sort by key gives each u its in-edges in step order at [in_off[u], in_off[u + 1]).  A warp per vertex v.
__global__ void __launch_bounds__(256) k_as_step_keys(int64_t n, const int32_t *__restrict__ off,
                                                      const int32_t *__restrict__ adj, const int32_t *__restrict__ inv,
                                                      u64 *keys, int32_t *pos) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t v = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < n; v += nwarps) {
		const u64 orig = (u64)(uint32_t)inv[v];
		for (int e = off[v] + lane; e < off[v + 1]; e += 32) {
			keys[e] = (u64)(uint32_t)adj[e] * (u64)n + orig;
			pos[e] = e;
		}
	}
}

// The lists of the batch's rows: a block per row (grid-stride), a warp per rank (see the top).  List r of a row goes
// to walk[slot_off[row] + r * len]: [s, e1, v1, ..., eh, t] in original vertex ids and edge rowids.
__global__ void k_as_unrank(int b0, int L, int64_t n, const int32_t *__restrict__ batch_rows,
                                                   const int *__restrict__ batch_n,
                                                   const int32_t *__restrict__ row_lane,
                                                   const int32_t *__restrict__ pdst, const int64_t *__restrict__ dst,
                                                   const uint16_t *__restrict__ level,
                                                   const int64_t *__restrict__ sigma, const int32_t *__restrict__ in_off,
                                                   const u64 *__restrict__ step_key, const int32_t *__restrict__ step_pos,
                                                   const int32_t *__restrict__ perm, const int64_t *__restrict__ edge_ids,
                                                   const int64_t *__restrict__ npaths, const int64_t *__restrict__ plen,
                                                   const int64_t *__restrict__ out_lengths,
                                                   const int64_t *__restrict__ slot_off, int64_t *walk) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
	const int nb = *batch_n;
	for (int j = blockIdx.x; j < nb; j += gridDim.x) {
		const int row = batch_rows[j];
		if (out_lengths[row] <= 1) {
			continue; // NULL, or [src] (k_path_trivial)
		}
		const int l = row_lane[row] - b0;
		const int64_t len = plen[row], np = npaths[row];
		int64_t *base = walk + slot_off[row];
		for (int64_t rank = warp; rank < np; rank += nw) {
			int64_t *out = base + rank * len;
			u64 r = (u64)rank;
			int cur = pdst[row];
			if (lane == 0) {
				out[len - 1] = dst[row];
			}
			for (int k = (int)((len - 1) / 2); k >= 1; k--) {
				const uint16_t hp = (uint16_t)(k - 1);
				const int e1 = in_off[cur + 1];
				const u64 key0 = (u64)(uint32_t)cur * (u64)n;
				int pick_orig = -1, pick_pos = -1;
				for (int c = in_off[cur]; c < e1 && pick_pos < 0; c += 32) {
					const int e = c + lane;
					u64 sg = 0;
					int orig = 0, pos = 0;
					if (e < e1) {
						orig = (int)(step_key[e] - key0);
						pos = step_pos[e];
						const int64_t cell = (int64_t)perm[orig] * L + l;
						if (level[cell] == hp) {
							sg = hp == 0 ? 1ull : (u64)sigma[cell];
						}
					}
					u64 incl = sg;
#pragma unroll
					for (int d = 1; d < 32; d <<= 1) {
						const u64 t = __shfl_up_sync(FULL_MASK, incl, d);
						if (lane >= d) {
							incl = sat_add(incl, t);
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
					break; // (cannot happen while the premise at the top holds: sigma(cur) > r)
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

// The hook of both functions (see the top)
struct AllShortest : PathHook {
	pgq_csr *csr;
	int64_t max_paths;
	int64_t *count, *npaths, *plen;
	u64 *ctr;
	const int64_t *d_dst;
	const u64 *step_key = nullptr; // all_shortest_paths: the step lists
	const int32_t *step_pos = nullptr;
	int batch(const PathBatch &b) override {
		cudaStream_t s = b.s;
		const int64_t n_ab = csr->n_ab;
		const int sms = csr->ctx->sm_count;
		int64_t *sigma;
		PGQ_TRY(pgq_ws_reserve(b.ws, WS_AS_SIGMA, (size_t)std::max<int64_t>(n_ab, 1) * b.L * sizeof(int64_t),
		                       (void **)&sigma));
		PGQ_CUDA(cudaMemsetAsync(&ctr[AS_K], 0, sizeof(u64), s));
		const unsigned row_grid = grid_size((b.rows_ub + 255) / 256, (int64_t)sms * 8);
		k_as_depth<<<row_grid, 256, 0, s>>>(b.b0, b.L, b.batch_rows, b.batch_n, b.row_lane, b.pdst, b.level, ctr);
		PGQ_CUDA(cudaGetLastError());
		u64 h_ctr[3] = {0, 0, 0};
		PGQ_CUDA(cudaMemcpyAsync(h_ctr, ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		const int K = (int)h_ctr[AS_K];
		for (int k = 1; k <= K; k++) {
			k_sigma_level<<<grid_size((n_ab + 7) / 8, (int64_t)sms * 8), 256, 0, s>>>(k, n_ab, b.L, csr->in.off, csr->in.adj,
			                                                                      b.level, sigma);
		}
		k_as_rows<<<row_grid, 256, 0, s>>>(b.b0, b.L, b.batch_rows, b.batch_n, b.row_lane, b.psrc, b.pdst, b.level, sigma,
		                                   max_paths, lists ? 1 : 0, count, npaths, plen, b.out_lengths, b.slot_off, ctr);
		PGQ_CUDA(cudaGetLastError());
		b.st->kernel_launches += 2 + K;
		if (!lists) {
			return PGQ_OK;
		}
		PGQ_CUDA(cudaMemcpyAsync(h_ctr, ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		if (h_ctr[AS_SATURATED]) {
			return pgq_fail(PGQ_ERR_UNSUPPORTED, "a row has INT64_MAX or more shortest paths: max_paths = 0 cannot list them");
		}
		// (the rows without a lane add at most one element each behind the last batch)
		const u64 total = h_ctr[AS_TOTAL];
		if (total > (AS_MAX / sizeof(int64_t)) - (u64)csr->n - (u64)0x7fffffff) {
			return pgq_fail(PGQ_ERR_OOM, "the shortest paths of one call hold too many elements (%llu)",
			                (unsigned long long)total);
		}
		int64_t *walk;
		PGQ_TRY(pgq_ws_grow(b.ws, WS_WALK, (size_t)total * sizeof(int64_t), (size_t)*b.walk_bound * sizeof(int64_t), s,
		                    (void **)&walk));
		*b.walk_bound = (int64_t)total;
		k_as_unrank<<<grid_size(b.rows_ub, (int64_t)sms * 16), 256, 0, s>>>(
		    b.b0, b.L, csr->n, b.batch_rows, b.batch_n, b.row_lane, b.pdst, d_dst, b.level, sigma, csr->in.off, step_key,
		    step_pos, csr->perm, csr->edge_ids, npaths, plen, b.out_lengths, b.slot_off, walk);
		PGQ_CUDA(cudaGetLastError());
		b.st->kernel_launches++;
		return PGQ_OK;
	}
};

// The step lists of the CSR (k_as_step_keys + radix_sort_pairs) into the workspace
int build_step_lists(pgq_csr *csr, Workspace *ws, cudaStream_t s, const u64 **keys, const int32_t **pos,
                     int64_t *launches) {
	const int64_t n = csr->n, m = csr->m;
	const size_t cells = (size_t)std::max<int64_t>(m, 1);
	uint64_t *ka, *kb;
	int32_t *pa, *pb;
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_STEP_KEY_A, cells * sizeof(u64), (void **)&ka));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_STEP_KEY_B, cells * sizeof(u64), (void **)&kb));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_STEP_POS_A, cells * sizeof(int32_t), (void **)&pa));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_STEP_POS_B, cells * sizeof(int32_t), (void **)&pb));
	*keys = reinterpret_cast<const u64 *>(ka);
	*pos = pa;
	if (m == 0) {
		return PGQ_OK;
	}
	k_as_step_keys<<<grid_size((n + 7) / 8, (int64_t)csr->ctx->sm_count * 16), 256, 0, s>>>(
	    n, csr->out.off, csr->out.adj, csr->inv, reinterpret_cast<u64 *>(ka), pa);
	PGQ_CUDA(cudaGetLastError());
	int end_bit = 1;
	while (end_bit < 64 && ((u64)1 << end_bit) < (u64)n * (u64)n) {
		end_bit++;
	}
	uint64_t *kres;
	int32_t *pres;
	PGQ_TRY(radix_sort_pairs(ws, ka, kb, pa, pb, m, end_bit, s, &kres, &pres));
	*keys = reinterpret_cast<const u64 *>(kres);
	*pos = pres;
	(*launches)++; // (radix_sort_pairs' own launches are not counted)
	return PGQ_OK;
}

// Both entry points: lists = false is shortest_path_count (max_paths, the list outputs unused)
static int all_shortest(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                        const uint8_t *dst_valid, const pgq_options *opts, bool lists, int64_t max_paths,
                        int64_t *out_count, int64_t *out_npaths, int64_t *out_path_len, int64_t *out_offsets,
                        uint8_t *out_valid, int64_t **out_elems, int64_t *out_total, pgq_stats *stats) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (lists && (!out_elems || !out_total)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	if (lists) {
		*out_elems = nullptr;
		*out_total = 0;
	}
	if (p < 0 || (p > 0 && (!src || !dst))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (p > 0 && (!out_count || !out_valid || (lists && (!out_npaths || !out_path_len || !out_offsets)))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	if (max_paths < 0) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "max_paths must be >= 0 (0 = every path)");
	}
	if (p >= 0x7fffffffLL) {
		return pgq_fail(PGQ_ERR_RANGE, "too many pairs in one call");
	}
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	if (opts && opts->shard_count > 1) {
		return pgq_fail(PGQ_ERR_UNSUPPORTED, "shortest_path_count and all_shortest_paths have no multi-GPU form");
	}
	if (p == 0) {
		if (stats) {
			memset(stats, 0, sizeof(*stats));
		}
		return PGQ_OK;
	}
	// a row searches only when both of its ids are valid: a NULL destination folds into a NULL source
	std::vector<uint8_t> valid;
	if (src_valid || dst_valid) {
		valid.resize((size_t)p);
		for (int64_t i = 0; i < p; i++) {
			valid[(size_t)i] = (!src_valid || src_valid[i]) && (!dst_valid || dst_valid[i]) ? 1 : 0;
		}
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	const int64_t *d_src, *d_dst;
	const uint8_t *d_valid;
	int64_t *d_off, *d_lens;
	uint8_t *d_ov;
	AllShortest hook;
	hook.lists = lists;
	hook.csr = csr;
	hook.max_paths = max_paths;
	PGQ_TRY(stage_column(ws, WS_IN_SRC, src, b8, (const void **)&d_src));
	PGQ_TRY(stage_column(ws, WS_IN_DST, dst, b8, (const void **)&d_dst));
	PGQ_TRY(stage_column(ws, WS_IN_VALID, valid.empty() ? nullptr : valid.data(), (size_t)p, (const void **)&d_valid));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_VALID, (size_t)p, (void **)&d_ov));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_OFFSETS, b8, (void **)&d_off));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LENGTHS, b8, (void **)&d_lens));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_COUNT, b8, (void **)&hook.count));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_NPATHS, b8, (void **)&hook.npaths));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_PATH_LEN, b8, (void **)&hook.plen));
	PGQ_TRY(pgq_ws_reserve(ws, WS_AS_COUNTERS, 256, (void **)&hook.ctr));
	hook.d_dst = d_dst;
	// (the driver times itself from its own start: the work before it is timed here and added)
	PGQ_CUDA(cudaEventRecord(ws->ev_begin, s));
	PGQ_CUDA(cudaMemsetAsync(hook.ctr, 0, 256, s));
	k_as_init_rows<<<grid_size((p + 255) / 256, 4096), 256, 0, s>>>(p, d_src, d_dst, d_valid, hook.count, hook.npaths,
	                                                            hook.plen);
	PGQ_CUDA(cudaGetLastError());
	int64_t pre_launches = 1;
	if (lists) {
		PGQ_TRY(build_step_lists(csr, ws, s, &hook.step_key, &hook.step_pos, &pre_launches));
	}
	PGQ_CUDA(cudaEventRecord(ws->ev_end, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	float pre_ms = 0.f;
	PGQ_CUDA(cudaEventElapsedTime(&pre_ms, ws->ev_begin, ws->ev_end));
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	int64_t *d_elems = nullptr;
	int64_t total = 0;
	PGQ_TRY(pgq_bfs_paths_hooked(csr, ws, p, d_src, d_dst, d_valid, opts, d_off, d_lens, d_ov, &d_elems, &total, &hook,
	                             s, &st));
	st.kernel_launches += pre_launches;
	st.total_ms += pre_ms;
	int64_t *h_elems = nullptr;
	if (lists) {
		h_elems = (int64_t *)malloc((size_t)(total > 0 ? total : 1) * sizeof(int64_t));
		if (!h_elems) {
			return pgq_fail(PGQ_ERR_OOM, "host allocation of %lld path elements failed", (long long)total);
		}
	}
	cudaError_t e = cudaMemcpyAsync(out_count, hook.count, b8, cudaMemcpyDeviceToHost, s);
	if (lists) {
		if (e == cudaSuccess && total > 0) {
			e = cudaMemcpyAsync(h_elems, d_elems, (size_t)total * sizeof(int64_t), cudaMemcpyDeviceToHost, s);
		}
		if (e == cudaSuccess) e = cudaMemcpyAsync(out_npaths, hook.npaths, b8, cudaMemcpyDeviceToHost, s);
		if (e == cudaSuccess) e = cudaMemcpyAsync(out_path_len, hook.plen, b8, cudaMemcpyDeviceToHost, s);
		if (e == cudaSuccess) e = cudaMemcpyAsync(out_offsets, d_off, b8, cudaMemcpyDeviceToHost, s);
	}
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	g.settled = (e == cudaSuccess);
	if (e != cudaSuccess) {
		cudaGetLastError();
		free(h_elems);
		return pgq_fail(PGQ_ERR_CUDA, "copying shortest paths back failed: %s", cudaGetErrorString(e));
	}
	for (int64_t i = 0; i < p; i++) {
		out_valid[i] = out_count[i] > 0; // (a valid row has at least one path)
	}
	st.h2d_bytes += 2 * (int64_t)b8 + (valid.empty() ? 0 : p);
	st.d2h_bytes += lists ? 4 * (int64_t)b8 + total * (int64_t)sizeof(int64_t) : (int64_t)b8;
	if (lists) {
		*out_elems = h_elems;
		*out_total = total;
	}
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_shortest_path_count(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                                       const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                       int64_t *out_count, uint8_t *out_valid, pgq_stats *stats) {
	return all_shortest(csr, n_pairs, src, dst, src_valid, dst_valid, opts, false, 0, out_count, nullptr, nullptr,
	                    nullptr, out_valid, nullptr, nullptr, stats);
}

extern "C" int pgq_all_shortest_paths(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                                      const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                      int64_t max_paths, int64_t *out_count, int64_t *out_npaths, int64_t *out_path_len,
                                      int64_t *out_offsets, uint8_t *out_valid, int64_t **out_elems,
                                      int64_t *out_total, pgq_stats *stats) {
	return all_shortest(csr, n_pairs, src, dst, src_valid, dst_valid, opts, true, max_paths, out_count, out_npaths,
	                    out_path_len, out_offsets, out_valid, out_elems, out_total, stats);
}
