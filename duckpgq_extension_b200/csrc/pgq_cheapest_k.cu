// pgq_cheapest_k.cu -- cheapest_k_paths on the weighted device CSR: the k cheapest paths of a row in SQL/PGQ's WALK,
// TRAIL, ACYCLIC and SIMPLE path modes (SQL/PGQ's CHEAPEST k).  No reference function.  sm_90a only.
//
// The rounds are shortest_k_paths_mode's (km_run, pgq_kpaths_modes.cu's top), with the pool keyed (cost, h, steps) and
// WALK spurring like TRAIL at dev <= j <= L with no bans beyond D.  A spur search at j from u = P[j] with root R is one
// lane of a batched Bellman-Ford over weights >= 0 (a CSR with a weight below zero is refused before any work):
//   * seed (k_ck_seed): u has no distance of its own; each admissible first edge e = u -> x sets d(x) = min(cost(R) +
//     w(e)), which covers the closed spurs (u == t) with no special case.  The same kernel loads the lane's banned
//     vertices into its mask and TRAIL's root edges into the ban bitmap.  A spur with no admissible seed -- km_first_ok
//     and a sum below the sentinel, not NaN (k_ck_has_seed) -- takes no lane.
//   * sweeps: k_bf_sweep over the filter CkEdges, which skips each lane's banned vertices and edges and, for BIGINT, a
//     sum that would reach the sentinel (w >= sentinel - d, so nothing overflows).  A DOUBLE sum at or above the
//     sentinel never beats a slot (no slot is above it), and k_bf_sweep skips a NaN sum.  Seeding at cost(R) rather than
//     0 makes the fixed point the least cost of R + spur itself: addition rounded to nearest is monotone.
//   * tight BFS: level 1 is the seeds x with cost(R) + w(e) == d(x) (k_ck_tight_seed); level lv + 1 the heads without a
//     level of the lane's tight, unbanned edges v -> x out of level lv, d(v) + w == d(x) compared as values with the sum
//     below the sentinel (k_ck_tight_level, a warp per frontier vertex as in k_bf_sweep).  A batch expands while a lane
//     that has not levelled its target grew at the last level (k_ck_finish).
//   * walk back (k_ck_walk, k_km_walk's with the tight test): from t over the step lists, at level >= 2 the first entry
//     whose parent has level - 1 and whose edge is tight and not banned; at level 1 the first admissible tight position
//     of u's adjacency.  It needs no parent key per (vertex, lane).
// The spur so found is the least admissible one by (cost, h, steps from t back to u), and R + spur the least path of its
// Lawler class; DESIGN.md §3 has the argument.
#include <algorithm>
#include <cstring>
#include <vector>

#include "pgq_bf.cuh"
#include "pgq_count.cuh"
#include "pgq_kpaths.cuh"
#include "pgq_tile.cuh"

#define CK_BUDGET ((int64_t)2 << 30)
#define CK_UNSET 0xFFFFu   // no tight level; a level is at most 0xFFFE
#define CK_LEVEL_MAX 0xFFFE

// the distance key of a raw cost (a root's)
template <bool F64>
__device__ __forceinline__ u64 ck_key(int64_t bits) {
	return F64 ? f64_key(__longlong_as_double(bits)) : (u64)bits;
}

// the sum of the distance dk and weight bits w in the weight type's arithmetic, as a key in *nk; false when it is NaN
// or reaches the sentinel (for BIGINT tested before the addition: d <= sentinel and w >= 0)
template <bool F64>
__device__ __forceinline__ bool ck_sum(u64 dk, int64_t w, u64 *nk) {
	if (F64) {
		const double c = key_f64(dk) + __longlong_as_double(w);
		*nk = f64_key(c);
		return c < BF_INF_F64;
	}
	*nk = dk + (u64)w;
	return w < BF_INF_I64 - (long long)dk;
}

// two distance keys hold equal values (-0.0 == 0.0)
template <bool F64>
__device__ __forceinline__ bool ck_eq(u64 a, u64 b) {
	return F64 ? key_f64(a) == key_f64(b) : a == b;
}

// The spur searches' edge filter for k_bf_sweep (pgq_bf.cuh): lane l of the batch admits the edge at out-CSR position e
// into x unless x is one of its banned vertices or e one of its banned positions (ban_bits null: none), and for BIGINT
// only while the sum stays below the sentinel.
template <bool F64>
struct CkEdges {
	int wd;
	const u64 *vban;
	const uint32_t *ban_bits;
	const int64_t *keys;
	int64_t nkeys;
	__device__ __forceinline__ bool banned(int64_t e, int x, int l) const {
		return ((vban[(int64_t)x * wd + (l >> 6)] >> (l & 63)) & 1) ||
		       (ban_bits && ((ban_bits[e >> 5] >> (e & 31)) & 1) && ((km_ban_mask(keys, nkeys, e, l >> 6) >> (l & 63)) & 1));
	}
	__device__ __forceinline__ bool edge(int64_t e, int u, int l, u64 dk, int64_t w) const {
		return (F64 || w < BF_INF_I64 - (long long)dk) && !banned(e, u, l);
	}
};

// whether each spur of a round has an admissible seed: a warp per spur
template <bool F64>
__global__ void __launch_bounds__(256) k_ck_has_seed(int64_t ns, const KmSpur *__restrict__ spurs,
                                                     const int32_t *__restrict__ lists, const int64_t *__restrict__ root,
                                                     const int32_t *__restrict__ out_off,
                                                     const int32_t *__restrict__ out_adj,
                                                     const int64_t *__restrict__ w_bits, uint8_t *has) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < ns; i += nwarps) {
		const KmSpur sp = spurs[i];
		const u64 rk = ck_key<F64>(root[i]);
		const int e1 = out_off[sp.u + 1];
		bool any = false;
		for (int c = out_off[sp.u]; c < e1 && !any; c += 32) {
			const int e = c + lane;
			u64 nk;
			any = __any_sync(FULL_MASK, e < e1 && km_first_ok(sp, lists, e, out_adj[e]) && ck_sum<F64>(rk, w_bits[e], &nk));
		}
		if (lane == 0) {
			has[i] = any;
		}
	}
}

// The seeds of each lane (a warp per lane): its banned vertices into vban, TRAIL's banned positions into the bitmap
// (ban_bits nullable), and d(x) = min(cost(R) + w(e)) over u's admissible first edges e = u -> x, x dirty
template <bool F64>
__global__ void __launch_bounds__(256) k_ck_seed(int cnt, int wd, int W, const int32_t *__restrict__ lane_spur,
                                                 const KmSpur *__restrict__ spurs, const int32_t *__restrict__ lists,
                                                 const int64_t *__restrict__ root, const int32_t *__restrict__ out_off,
                                                 const int32_t *__restrict__ out_adj,
                                                 const int64_t *__restrict__ w_bits, u64 *vban, uint32_t *ban_bits,
                                                 u64 *dist, uint32_t *dirty) {
	const int lane = threadIdx.x & 31;
	const int nwarps = (gridDim.x * blockDim.x) >> 5;
	for (int l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < cnt; l += nwarps) {
		const int32_t x0 = lane_spur[l];
		const KmSpur sp = spurs[x0];
		const u64 rk = ck_key<F64>(root[x0]);
		const u64 bit = 1ull << (l & 63);
		for (int i = lane; i < sp.nvb; i += 32) {
			atomicOr(&vban[(int64_t)lists[sp.vb + i] * wd + (l >> 6)], bit);
		}
		if (ban_bits) {
			for (int i = lane; i < sp.neb; i += 32) {
				const int32_t e = lists[sp.eb + i];
				atomicOr(&ban_bits[e >> 5], 1u << (e & 31));
			}
		}
		const int e1 = out_off[sp.u + 1];
		for (int e = out_off[sp.u] + lane; e < e1; e += 32) {
			const int32_t x = out_adj[e];
			u64 nk;
			if (km_first_ok(sp, lists, e, x) && ck_sum<F64>(rk, w_bits[e], &nk)) {
				u64 *slot = &dist[(int64_t)x * W + l];
				if (F64) {
					atomicMin(slot, nk);
				} else {
					atomicMin(reinterpret_cast<long long *>(slot), (long long)nk);
				}
				atomicOr(&dirty[x >> 5], 1u << (x & 31));
			}
		}
	}
}

// Level 1 of each lane's tight BFS (a warp per lane): the seeds x of a tight admissible first edge, cost(R) + w(e) ==
// d(x), into the frontier; a lane with one is flagged in grew
template <bool F64>
__global__ void __launch_bounds__(256) k_ck_tight_seed(int cnt, int W, const int32_t *__restrict__ lane_spur,
                                                       const KmSpur *__restrict__ spurs, const int32_t *__restrict__ lists,
                                                       const int64_t *__restrict__ root,
                                                       const int32_t *__restrict__ out_off,
                                                       const int32_t *__restrict__ out_adj,
                                                       const int64_t *__restrict__ w_bits, const u64 *__restrict__ dist,
                                                       uint16_t *level, uint32_t *front, u64 *grew) {
	const int lane = threadIdx.x & 31;
	const int nwarps = (gridDim.x * blockDim.x) >> 5;
	for (int l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < cnt; l += nwarps) {
		const KmSpur sp = spurs[lane_spur[l]];
		const u64 rk = ck_key<F64>(root[lane_spur[l]]);
		const int e1 = out_off[sp.u + 1];
		bool any = false;
		for (int e = out_off[sp.u] + lane; e < e1; e += 32) {
			const int32_t x = out_adj[e];
			u64 nk;
			if (km_first_ok(sp, lists, e, x) && ck_sum<F64>(rk, w_bits[e], &nk) &&
			    ck_eq<F64>(nk, dist[(int64_t)x * W + l])) {
				level[(int64_t)x * W + l] = 1;
				atomicOr(&front[x >> 5], 1u << (x & 31));
				any = true;
			}
		}
		if (__any_sync(FULL_MASK, any) && lane == 0) {
			atomicOr(&grew[l >> 6], 1ull << (l & 63));
		}
	}
}

// After a level: a lane whose target has a level is done with spur length hlen = that level; a lane not done that grew
// counts as still searching (ctr).  grew is cleared for the next level.  One block.
__global__ void k_ck_finish(int cnt, int W, const int32_t *__restrict__ lane_spur, const KmSpur *__restrict__ spurs,
                            const uint16_t *__restrict__ level, u64 *grew, u64 *done, int32_t *hlen, int *ctr) {
	for (int l = threadIdx.x; l < cnt; l += blockDim.x) {
		const u64 bit = 1ull << (l & 63);
		if (done[l >> 6] & bit) {
			continue;
		}
		const uint16_t h = level[(int64_t)spurs[lane_spur[l]].t * W + l];
		if (h != CK_UNSET) {
			atomicOr(&done[l >> 6], bit);
			hlen[l] = h;
		} else if (grew[l >> 6] & bit) {
			atomicAdd(ctr, 1);
		}
	}
	__syncthreads(); // (every lane read grew before it is cleared)
	for (int j = threadIdx.x; j < (W + 63) / 64; j += blockDim.x) {
		grew[j] = 0;
	}
}

// One tight level: a warp per vertex of the frontier cur, 32 lanes at a time (k_bf_sweep's layout).  Each lane still
// searching with v at level lv passes lv + 1 along its tight, unbanned edges v -> x to the x without a level; x joins
// next and the lane is flagged in grew.
template <bool F64>
__global__ void __launch_bounds__(256) k_ck_tight_level(int lv, int64_t n, int W, const int32_t *__restrict__ off,
                                                        const int32_t *__restrict__ adj,
                                                        const int64_t *__restrict__ w_bits,
                                                        const u64 *__restrict__ dist, const u64 *__restrict__ done,
                                                        const CkEdges<F64> ban, uint16_t *level,
                                                        const uint32_t *__restrict__ cur, uint32_t *next, u64 *grew) {
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	const uint16_t hk = (uint16_t)lv, hk1 = (uint16_t)(lv + 1);
	for (int64_t v = warp; v < n; v += nwarps) {
		if (!(cur[v >> 5] & (1u << (v & 31)))) {
			continue;
		}
		const int e0 = off[v], e1 = off[v + 1];
		for (int g = 0; g < W; g += 32) {
			const int l = g + lane;
			const bool act = level[v * W + l] == hk && !((done[l >> 6] >> (l & 63)) & 1);
			if (!__any_sync(FULL_MASK, act)) {
				continue;
			}
			const u64 dk = dist[v * W + l];
			bool got = false;
			for (int e = e0; e < e1; e++) {
				const int x = adj[e];
				bool fresh = false;
				if (act) {
					const int64_t slot = (int64_t)x * W + l;
					u64 nk;
					if (level[slot] == CK_UNSET && ck_sum<F64>(dk, w_bits[e], &nk) && ck_eq<F64>(nk, dist[slot]) &&
					    !ban.banned(e, x, l)) {
						level[slot] = hk1;
						fresh = got = true;
					}
				}
				if (__any_sync(FULL_MASK, fresh) && lane == 0) {
					atomicOr(&next[x >> 5], 1u << (x & 31));
				}
			}
			const unsigned grown = __ballot_sync(FULL_MASK, got);
			if (grown && lane == 0) {
				atomicOr(&grew[g >> 6], (u64)grown << (g & 63));
			}
		}
	}
}

// The spurs of a batch's found lanes, a warp per lane (see the top): step i of lane l (0 = the edge out of u) goes to
// steps[lane_off[l] + i] as (parent's internal id, out-CSR position), to step_elems as (parent's original id, edge
// rowid) and to step_w as the edge's weight bits
template <bool F64>
__global__ void __launch_bounds__(256) k_ck_walk(int cnt, int W, int64_t n, const int32_t *__restrict__ lane_spur,
                                                 const KmSpur *__restrict__ spurs, const int32_t *__restrict__ lists,
                                                 const int64_t *__restrict__ root, const int32_t *__restrict__ hlen,
                                                 const int64_t *__restrict__ lane_off, const uint16_t *__restrict__ level,
                                                 const u64 *__restrict__ dist, const int32_t *__restrict__ in_off,
                                                 const u64 *__restrict__ step_key, const int32_t *__restrict__ step_pos,
                                                 const int32_t *__restrict__ perm, const int32_t *__restrict__ inv,
                                                 const int32_t *__restrict__ out_off, const int32_t *__restrict__ out_adj,
                                                 const int64_t *__restrict__ edge_ids,
                                                 const int64_t *__restrict__ w_bits, int2 *steps,
                                                 longlong2 *step_elems, int64_t *step_w) {
	const int lane = threadIdx.x & 31;
	const int nwarps = (gridDim.x * blockDim.x) >> 5;
	for (int l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < cnt; l += nwarps) {
		const int h = hlen[l];
		if (h == 0) {
			continue;
		}
		const KmSpur sp = spurs[lane_spur[l]];
		const int32_t *eb = lists + sp.eb;
		int2 *out = steps + lane_off[l];
		longlong2 *oel = step_elems + lane_off[l];
		int64_t *ow = step_w + lane_off[l];
		int cur = sp.t;
		for (int lv = h; lv >= 2; lv--) {
			const int e1 = in_off[cur + 1];
			const u64 key0 = (u64)(uint32_t)cur * (u64)n;
			const u64 dcur = dist[(int64_t)cur * W + l];
			int pick = -1;
			for (int c = in_off[cur]; c < e1 && pick < 0; c += 32) {
				const int e = c + lane;
				int orig = 0, pos = 0, par = 0;
				bool ok = false;
				if (e < e1) {
					orig = (int)(step_key[e] - key0);
					pos = step_pos[e];
					par = perm[orig];
					u64 nk;
					ok = level[(int64_t)par * W + l] == lv - 1 && !km_in(eb, sp.neb, pos) &&
					     ck_sum<F64>(dist[(int64_t)par * W + l], w_bits[pos], &nk) && ck_eq<F64>(nk, dcur);
				}
				const unsigned hit = __ballot_sync(FULL_MASK, ok);
				if (hit) {
					const int w = __ffs(hit) - 1;
					pick = __shfl_sync(FULL_MASK, par, w);
					pos = __shfl_sync(FULL_MASK, pos, w);
					orig = __shfl_sync(FULL_MASK, orig, w);
					if (lane == 0) {
						out[lv - 1] = make_int2(pick, pos);
						oel[lv - 1] = make_longlong2(orig, edge_ids[pos]);
						ow[lv - 1] = w_bits[pos];
					}
				}
			}
			if (pick < 0) {
				break; // (cannot happen: a vertex at level lv has a tight admissible parent at level lv - 1)
			}
			cur = pick;
		}
		const u64 rk = ck_key<F64>(root[lane_spur[l]]);
		const u64 dcur = dist[(int64_t)cur * W + l];
		const int e1 = out_off[sp.u + 1];
		for (int c = out_off[sp.u]; c < e1; c += 32) {
			const int e = c + lane;
			u64 nk;
			const bool ok = e < e1 && out_adj[e] == cur && km_first_ok(sp, lists, e, cur) &&
			                ck_sum<F64>(rk, w_bits[e], &nk) && ck_eq<F64>(nk, dcur);
			const unsigned hit = __ballot_sync(FULL_MASK, ok);
			if (hit) {
				const int w = __ffs(hit) - 1;
				if (lane == 0) {
					out[0] = make_int2(sp.u, c + w);
					oel[0] = make_longlong2(inv[sp.u], edge_ids[c + w]);
					ow[0] = w_bits[c + w];
				}
				break;
			}
		}
	}
}

// The Bellman-Ford spur search of cheapest_k_paths (see the top)
template <bool F64>
struct CkSearch : KmSearch {
	pgq_csr *csr;
	const u64 *step_key = nullptr;
	const int32_t *step_pos = nullptr;
	const int64_t *root = nullptr; // the round's root costs
	u64 *dist = nullptr, *vban = nullptr, *grew = nullptr, *done = nullptr;
	uint32_t *dirty = nullptr, *front = nullptr;
	uint16_t *level = nullptr;
	int *flags = nullptr; // [0] a sweep changed a distance, [1] lanes still searching
	// W: opts->lanes, or the widest of 256 .. 32 whose distance array n x W x 8 bytes fits 2 GiB (run_bf's rule)
	CkSearch(pgq_csr *c, const pgq_options *opts) : csr(c) {
		lane_min = 32;
		costs = true;
		cap = opts && opts->lanes ? opts->lanes : 256;
		while (!(opts && opts->lanes) && cap > 32 && std::max<int64_t>(c->n, 1) * cap * 8 > CK_BUDGET) {
			cap >>= 1;
		}
	}
	int begin(Workspace *ws, const u64 *sk, const int32_t *sp) override {
		const int64_t n = std::max<int64_t>(csr->n, 1);
		const size_t words = (size_t)n / 32 + 1;
		const int wd = (cap + 63) / 64;
		step_key = sk;
		step_pos = sp;
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_DIST, (size_t)n * cap * sizeof(u64), (void **)&dist));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_LEVEL, (size_t)n * cap * sizeof(uint16_t), (void **)&level));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_VBAN, (size_t)n * wd * sizeof(u64), (void **)&vban));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_DIRTY, words * sizeof(uint32_t), (void **)&dirty));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_FRONT, 2 * words * sizeof(uint32_t), (void **)&front));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_GREW, (size_t)wd * sizeof(u64), (void **)&grew));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_DONE, (size_t)wd * sizeof(u64), (void **)&done));
		PGQ_TRY(pgq_ws_reserve(ws, WS_CK_FLAGS, 256, (void **)&flags));
		return PGQ_OK;
	}
	int has_seed(Workspace *ws, int64_t ns, const KmSpur *spurs, const int32_t *lists, const std::vector<int64_t> &roots,
	             uint8_t *has, pgq_stats *st) override {
		PGQ_TRY(stage_column(ws, WS_CK_ROOT, roots.data(), roots.size() * sizeof(int64_t), (const void **)&root));
		st->h2d_bytes += (int64_t)(roots.size() * sizeof(int64_t));
		k_ck_has_seed<F64><<<grid_size((ns + 7) / 8, (int64_t)csr->ctx->sm_count * 16), 256, 0, ws->stream>>>(
		    ns, spurs, lists, root, csr->out.off, csr->out.adj, csr->w_bits, has);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches++;
		return PGQ_OK;
	}
	int search(Workspace *ws, const KmBatch &b, pgq_stats *st) override {
		cudaStream_t s = ws->stream;
		const int64_t n = csr->n;
		const int sms = csr->ctx->sm_count;
		const int W = b.W, wd = (W + 63) / 64, cnt = b.cnt;
		const size_t cells = (size_t)std::max<int64_t>(n, 1) * W;
		const size_t words = (size_t)n / 32 + 1;
		const unsigned vert_grid = grid_size((n + 7) / 8, (int64_t)sms * 8);
		k_bf_init<F64><<<grid_size(((int64_t)cells + 255) / 256, (int64_t)sms * 16), 256, 0, s>>>((int64_t)cells, dist);
		PGQ_CUDA(cudaMemsetAsync(vban, 0, (size_t)n * wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(dirty, 0, words * sizeof(uint32_t), s));
		PGQ_CUDA(cudaMemsetAsync(level, 0xff, cells * sizeof(uint16_t), s));
		PGQ_CUDA(cudaMemsetAsync(front, 0, 2 * words * sizeof(uint32_t), s));
		PGQ_CUDA(cudaMemsetAsync(grew, 0, (size_t)wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(done, 0, (size_t)wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(b.hlen, 0, (size_t)W * sizeof(int32_t), s));
		k_ck_seed<F64><<<b.lane_grid, 256, 0, s>>>(cnt, wd, W, b.lane_spur, b.spurs, b.lists, root, csr->out.off,
		                                           csr->out.adj, csr->w_bits, vban, b.ban_bits, dist, dirty);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches += 2;
		const CkEdges<F64> keep = {wd, vban, b.ban_bits, b.keys, b.nkeys};
		for (;;) {
			int changed = 0;
			PGQ_CUDA(cudaMemsetAsync(flags, 0, sizeof(int), s));
			k_bf_sweep<F64, CkEdges<F64>><<<vert_grid, 256, 0, s>>>(n, W, csr->out.off, csr->out.adj, csr->w_bits, dist,
			                                                       dirty, flags, keep);
			PGQ_CUDA(cudaGetLastError());
			PGQ_CUDA(cudaMemcpyAsync(&changed, flags, sizeof(int), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st->kernel_launches++;
			st->levels++;
			st->d2h_bytes += (int64_t)sizeof(int);
			if (!changed) {
				break;
			}
		}
		k_ck_tight_seed<F64><<<b.lane_grid, 256, 0, s>>>(cnt, W, b.lane_spur, b.spurs, b.lists, root, csr->out.off,
		                                                 csr->out.adj, csr->w_bits, dist, level, front, grew);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches++;
		uint32_t *cur = front, *next = front + words;
		for (int lv = 1;; lv++) {
			int active = 0;
			PGQ_CUDA(cudaMemsetAsync(flags + 1, 0, sizeof(int), s));
			k_ck_finish<<<1, 1024, 0, s>>>(cnt, W, b.lane_spur, b.spurs, level, grew, done, b.hlen, flags + 1);
			PGQ_CUDA(cudaGetLastError());
			PGQ_CUDA(cudaMemcpyAsync(&active, flags + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st->kernel_launches++;
			st->d2h_bytes += (int64_t)sizeof(int);
			if (!active) {
				break;
			}
			if (lv + 1 > CK_LEVEL_MAX) {
				return pgq_fail(PGQ_ERR_UNSUPPORTED, "a spur search went beyond %d tight levels", CK_LEVEL_MAX);
			}
			PGQ_CUDA(cudaMemsetAsync(next, 0, words * sizeof(uint32_t), s));
			k_ck_tight_level<F64><<<vert_grid, 256, 0, s>>>(lv, n, W, csr->out.off, csr->out.adj, csr->w_bits, dist, done,
			                                                keep, level, cur, next, grew);
			PGQ_CUDA(cudaGetLastError());
			st->kernel_launches++;
			st->push_levels++;
			std::swap(cur, next);
		}
		PGQ_CUDA(cudaMemcpyAsync(b.h_hlen, b.hlen, (size_t)cnt * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		st->d2h_bytes += cnt * (int64_t)sizeof(int32_t);
		return PGQ_OK;
	}
	int walk(Workspace *ws, const KmBatch &b, const int64_t *lane_off, int2 *steps, longlong2 *step_elems,
	         int64_t *step_w, pgq_stats *st) override {
		k_ck_walk<F64><<<b.lane_grid, 256, 0, ws->stream>>>(
		    b.cnt, b.W, csr->n, b.lane_spur, b.spurs, b.lists, root, b.hlen, lane_off, level, dist, csr->in.off, step_key,
		    step_pos, csr->perm, csr->inv, csr->out.off, csr->out.adj, csr->edge_ids, csr->w_bits, steps, step_elems,
		    step_w);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches++;
		return PGQ_OK;
	}
};

extern "C" int pgq_cheapest_k_paths(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                    const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                    int64_t k, int32_t path_mode, int64_t *out_npaths, int64_t *out_first_path,
                                    uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
                                    void **out_costs, int64_t *out_total_paths, pgq_stats *stats) {
	if (out_costs) {
		*out_costs = nullptr;
	}
	pgq_options o = {};
	if (opts) {
		o = *opts;
	}
	o.lanes = 0; // (this call's widths, 32 .. 256, are checked below)
	PGQ_TRY(ks_check_call(csr, p, src, dst, &o, k, out_npaths, out_first_path, out_valid, out_path_offsets, out_elems,
	                      out_total_paths));
	if (opts && opts->lanes != 0 && opts->lanes != 32 && opts->lanes != 64 && opts->lanes != 128 && opts->lanes != 256) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "lanes must be 0, 32, 64, 128 or 256");
	}
	if (path_mode != PGQ_PATH_WALK && path_mode != PGQ_PATH_TRAIL && path_mode != PGQ_PATH_ACYCLIC &&
	    path_mode != PGQ_PATH_SIMPLE) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "unknown path mode %d", (int)path_mode);
	}
	if (!csr->w_bits || csr->weight_type == 0) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing cheapest path");
	}
	if (csr->neg_weights) {
		return pgq_fail(PGQ_ERR_UNSUPPORTED, "cheapest_k_paths needs weights >= 0");
	}
	if (csr->weight_type == 2) {
		CkSearch<true> ck(csr, opts);
		return km_run(csr, p, src, dst, src_valid, dst_valid, opts, k, path_mode, nullptr, ck, out_npaths,
		              out_first_path, out_valid, out_path_offsets, out_elems, out_costs, out_total_paths, stats);
	}
	CkSearch<false> ck(csr, opts);
	return km_run(csr, p, src, dst, src_valid, dst_valid, opts, k, path_mode, nullptr, ck, out_npaths, out_first_path,
	              out_valid, out_path_offsets, out_elems, out_costs, out_total_paths, stats);
}
