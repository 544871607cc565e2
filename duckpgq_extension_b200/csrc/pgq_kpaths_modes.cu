// pgq_kpaths_modes.cu -- shortest_k_paths in SQL/PGQ's TRAIL, ACYCLIC and SIMPLE path modes on the device CSR (the
// reference parses the modes and rejects all but WALK).  No reference function.  sm_90a only.
//
// Yen's algorithm with Lawler's rule, one row's paths at a time per round, every row of a round at once:
//   * each row keeps A, its accepted paths (each with the spur index dev it deviated at), and a de-duplicated
//     candidate pool ordered like the result.  Round 0 searches from s with no bans (s == t: A[0] = [s], no search);
//     every later round spurs off the path P the row accepted last, at each j of its mode's range (see the header),
//     then each live row moves its pool's minimum into A.  A row stops with k paths or an empty pool.
//   * a spur search at j is a BFS from u = P[j] with root R = P's first j steps: D (edge j of every accepted path
//     through R) restricts its first edge, the root's vertices are banned (ACYCLIC, SIMPLE; t exempt for SIMPLE at
//     s == t), the root's edges are banned at every level (TRAIL).  u has no level 0: level 1 is every out-neighbour
//     of u through an entry that is not in D, not banned and does not lead to a banned vertex, and t is found when it
//     gets a level >= 1, which covers the closed spurs (u == t) with no special case.
//   * the searches of a round take lanes in (row, j) order, W per batch; a spur with no admissible first edge takes
//     none (k_km_has_seed decides it before the round is packed).  Per batch: k_km_seed pre-loads each lane's bans
//     into its seen bits (and TRAIL's root edges into a bitmap over out-CSR positions with a sorted (position, lane)
//     table), expands u's adjacency into level 1; k_km_level pushes the frontier one level over the out-CSR, a thread
//     per position; k_km_fold folds the level in and k_km_finish marks the lanes whose t has a bit, one sync a level,
//     until no lane that has not reached t has a frontier.  k_km_walk then walks each found spur back from t over the
//     step lists (build_step_lists, shared with all_shortest_paths and shortest_k_paths): at level >= 2 the first
//     entry whose parent has level - 1 and whose edge is not banned, at level 1 the first position of u's adjacency
//     to the vertex that is not in D and not banned.  The host appends R + spur to the row's pool unless it is known.
//   * the walk back's choices give the first spur in the result's order among the shortest admissible ones, and
//     Lawler's rule (spurs only at j >= dev) with D gives each candidate once; DESIGN.md §3 has the argument,
//     including why TRAIL also spurs at j = len(P), past t.
// The BFS drivers' WS_SEEN / WS_VISIT_* are not touched: the searches have masks of their own (WS_KM_*).
// shortest_k_groups in these modes runs the same rounds (km_run) with another stop test before a row accepts its pool's
// least path: an empty pool, k groups and a longer least path, or max_paths paths listed (DESIGN.md §3).
#include <algorithm>
#include <cstring>
#include <map>
#include <set>
#include <vector>

#include "pgq_count.cuh"
#include "pgq_kpaths.cuh"
#include "pgq_tile.cuh"

#define KM_BUDGET ((int64_t)4 << 30)

// The batch's counters: [0] lanes still searching; [1] a lane reached a level beyond KM_PATH_MAX
enum { KM_ACTIVE = 0, KM_TOO_LONG = 1 };

// internal ids of the rows' sources and targets
__global__ void k_km_ids(int64_t cnt, const int64_t *__restrict__ ids, const int32_t *__restrict__ perm, int32_t *pids) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (int64_t)gridDim.x * blockDim.x) {
		pids[i] = perm[ids[i]];
	}
}

// whether each spur of a round has an admissible first edge: a warp per spur
__global__ void __launch_bounds__(256) k_km_has_seed(int64_t ns, const KmSpur *__restrict__ spurs,
                                                     const int32_t *__restrict__ lists, const int32_t *__restrict__ out_off,
                                                     const int32_t *__restrict__ out_adj, uint8_t *has) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < ns; i += nwarps) {
		const KmSpur sp = spurs[i];
		const int e1 = out_off[sp.u + 1];
		bool any = false;
		for (int c = out_off[sp.u]; c < e1 && !any; c += 32) {
			const int e = c + lane;
			any = __any_sync(FULL_MASK, e < e1 && km_first_ok(sp, lists, e, out_adj[e]));
		}
		if (lane == 0) {
			has[i] = any;
		}
	}
}

// Level 1 of each lane (a warp per lane): the banned vertices' seen bits, TRAIL's banned positions into the bitmap
// (ban_bits nullable), u's admissible out-neighbours into the frontier at level 1
__global__ void __launch_bounds__(256) k_km_seed(int cnt, int wd, int W, const int32_t *__restrict__ lane_spur,
                                                 const KmSpur *__restrict__ spurs, const int32_t *__restrict__ lists,
                                                 const int32_t *__restrict__ out_off, const int32_t *__restrict__ out_adj,
                                                 u64 *seen, u64 *front, u64 *grew, uint16_t *level, uint32_t *ban_bits) {
	const int lane = threadIdx.x & 31;
	const int nwarps = (gridDim.x * blockDim.x) >> 5;
	for (int l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < cnt; l += nwarps) {
		const KmSpur sp = spurs[lane_spur[l]];
		const int word = l >> 6;
		const u64 bit = 1ull << (l & 63);
		for (int i = lane; i < sp.nvb; i += 32) {
			atomicOr(&seen[(int64_t)lists[sp.vb + i] * wd + word], bit);
		}
		if (ban_bits) {
			for (int i = lane; i < sp.neb; i += 32) {
				const int32_t e = lists[sp.eb + i];
				atomicOr(&ban_bits[e >> 5], 1u << (e & 31));
			}
		}
		const int e1 = out_off[sp.u + 1];
		bool any = false;
		for (int e = out_off[sp.u] + lane; e < e1; e += 32) {
			const int32_t v = out_adj[e];
			if (km_first_ok(sp, lists, e, v)) {
				atomicOr(&seen[(int64_t)v * wd + word], bit);
				atomicOr(&front[(int64_t)v * wd + word], bit);
				level[(int64_t)v * W + l] = 1;
				any = true;
			}
		}
		if (__any_sync(FULL_MASK, any) && lane == 0) {
			atomicOr(&grew[word], bit);
		}
	}
}

// One forward level over the out-CSR: every out-edge r -> x passes r's frontier bits of the lanes still searching to
// x, minus x's seen bits and minus the lanes that ban the position (ban_bits nullable).  A thread per out-CSR
// position; a warp finds the row of its first position by bisection (rows may be empty) and each thread walks on.
__global__ void __launch_bounds__(256) k_km_level(int64_t m, int64_t n, int wd, const int32_t *__restrict__ out_off,
                                                  const int32_t *__restrict__ out_adj, const u64 *__restrict__ front,
                                                  const u64 *__restrict__ seen, const u64 *__restrict__ done,
                                                  const uint32_t *__restrict__ ban_bits,
                                                  const int64_t *__restrict__ ban_keys, int64_t nkeys, u64 *next) {
	const int lane = threadIdx.x & 31;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	for (int64_t base = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; base < m; base += nwarps * 32) {
		int64_t lo = 0, hi = n - 1; // the first row r with out_off[r + 1] > base
		while (lo < hi) {
			const int64_t mid = (lo + hi) >> 1;
			if (out_off[mid + 1] > base) {
				hi = mid;
			} else {
				lo = mid + 1;
			}
		}
		const int64_t e = base + lane;
		if (e >= m) {
			continue;
		}
		int64_t r = lo;
		while (out_off[r + 1] <= e) {
			r++;
		}
		const int64_t x = out_adj[e];
		const bool banned = ban_bits && ((ban_bits[e >> 5] >> (e & 31)) & 1);
		for (int j = 0; j < wd; j++) {
			const u64 f = front[r * wd + j] & ~done[j];
			if (f) {
				u64 nb = f & ~seen[x * wd + j];
				if (nb && banned) {
					nb &= ~km_ban_mask(ban_keys, nkeys, e, j);
				}
				if (nb) {
					atomicOr(&next[x * wd + j], nb);
				}
			}
		}
	}
}

// folds level lv in: the new bits become seen, the frontier and the level; each lane that got one is flagged in grew
__global__ void __launch_bounds__(256) k_km_fold(int64_t n, int wd, int W, int lv, u64 *seen, u64 *front, u64 *next,
                                                 u64 *grew, uint16_t *level, u64 *ctr) {
	const int lane = threadIdx.x & 31;
	const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
	for (int64_t v0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ll; v0 < n; v0 += nthreads) {
		const int64_t v = v0 + lane;
		for (int j = 0; j < wd; j++) {
			u64 nw = 0;
			if (v < n) {
				const int64_t i = v * wd + j;
				nw = next[i] & ~seen[i];
				next[i] = 0;
				seen[i] |= nw;
				front[i] = nw;
				for (u64 b = nw; b; b &= b - 1) {
					level[v * W + j * 64 + __ffsll((long long)b) - 1] = (uint16_t)lv;
				}
			}
			const unsigned lo = __reduce_or_sync(FULL_MASK, (unsigned)nw);
			const unsigned hi = __reduce_or_sync(FULL_MASK, (unsigned)(nw >> 32));
			if (lane == 0 && (lo | hi)) {
				atomicOr(&grew[j], (u64)lo | ((u64)hi << 32));
				if (lv > KM_PATH_MAX) {
					ctr[KM_TOO_LONG] = 1;
				}
			}
		}
	}
}

// After a level: a lane whose t has a bit is done with spur length hlen = t's level; a lane not done that grew counts
// as still searching.  grew is cleared for the next level.
__global__ void k_km_finish(int cnt, int wd, int W, const int32_t *__restrict__ lane_spur,
                            const KmSpur *__restrict__ spurs, const u64 *__restrict__ seen,
                            const uint16_t *__restrict__ level, u64 *grew, u64 *done, int32_t *hlen, u64 *ctr) {
	for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < cnt; l += gridDim.x * blockDim.x) {
		const int word = l >> 6;
		const u64 bit = 1ull << (l & 63);
		if (done[word] & bit) {
			continue;
		}
		const int64_t t = spurs[lane_spur[l]].t;
		if (seen[t * wd + word] & bit) {
			atomicOr(&done[word], bit);
			hlen[l] = level[t * W + l];
		} else if (grew[word] & bit) {
			atomicAdd(&ctr[KM_ACTIVE], 1ull);
		}
	}
	__syncthreads(); // (one block: every lane read grew before it is cleared)
	for (int j = threadIdx.x; j < wd; j += blockDim.x) {
		grew[j] = 0;
	}
}

// The spurs of a batch's found lanes, a warp per lane (see the top): step i of lane l (0 = the edge out of u) goes to
// steps[lane_off[l] + i] as (parent's internal id, out-CSR position) and to step_elems as (parent's original id, edge
// rowid)
__global__ void __launch_bounds__(256) k_km_walk(int cnt, int W, int64_t n, const int32_t *__restrict__ lane_spur,
                                                 const KmSpur *__restrict__ spurs, const int32_t *__restrict__ lists,
                                                 const int32_t *__restrict__ hlen, const int64_t *__restrict__ lane_off,
                                                 const uint16_t *__restrict__ level, const int32_t *__restrict__ in_off,
                                                 const u64 *__restrict__ step_key, const int32_t *__restrict__ step_pos,
                                                 const int32_t *__restrict__ perm, const int32_t *__restrict__ inv,
                                                 const int32_t *__restrict__ out_off, const int32_t *__restrict__ out_adj,
                                                 const int64_t *__restrict__ edge_ids, int2 *steps, longlong2 *step_elems) {
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
		int cur = sp.t;
		for (int lv = h; lv >= 2; lv--) {
			const int e1 = in_off[cur + 1];
			const u64 key0 = (u64)(uint32_t)cur * (u64)n;
			int pick = -1;
			for (int c = in_off[cur]; c < e1 && pick < 0; c += 32) {
				const int e = c + lane;
				int orig = 0, pos = 0, par = 0;
				bool ok = false;
				if (e < e1) {
					orig = (int)(step_key[e] - key0);
					pos = step_pos[e];
					par = perm[orig];
					ok = level[(int64_t)par * W + l] == lv - 1 && !km_in(eb, sp.neb, pos);
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
					}
				}
			}
			if (pick < 0) {
				break; // (cannot happen: a vertex at level lv has an admissible parent at level lv - 1)
			}
			cur = pick;
		}
		const int e1 = out_off[sp.u + 1];
		for (int c = out_off[sp.u]; c < e1; c += 32) {
			const int e = c + lane;
			const bool ok = e < e1 && out_adj[e] == cur && km_first_ok(sp, lists, e, cur);
			const unsigned hit = __ballot_sync(FULL_MASK, ok);
			if (hit) {
				const int w = __ffs(hit) - 1;
				if (lane == 0) {
					out[0] = make_int2(sp.u, c + w);
					oel[0] = make_longlong2(inv[sp.u], edge_ids[c + w]);
				}
				break;
			}
		}
	}
}

// a path of a row: its vertices (internal ids), out-CSR positions, elements [s, e1, v1, ..., t], the spur index it
// deviated at and, when its search has costs, the costs of its prefixes (cost[i]: its first i steps)
struct KmPath {
	std::vector<int32_t> v, pos;
	std::vector<int64_t> el, cost;
	int64_t dev = 0;
	int64_t h() const {
		return (int64_t)pos.size();
	}
	// (the cost when the search has costs, h, then the steps (parent's original id, position) from t back to s): the
	// result's order, and the identity of a path of the row.  A cost is >= 0 and never -0.0 (a sum from +0.0 of weights
	// >= 0), so its raw bits order as its value in both weight types.
	std::vector<int64_t> key(bool costs) const {
		std::vector<int64_t> k;
		k.reserve(2 * pos.size() + 2);
		if (costs) {
			k.push_back(cost.back());
		}
		k.push_back(h());
		for (int64_t i = h() - 1; i >= 0; i--) {
			k.push_back(el[2 * i]);
			k.push_back(pos[i]);
		}
		return k;
	}
};

struct KmRow {
	int64_t row;
	int32_t s, t;   // internal ids
	bool live = true;
	std::vector<KmPath> acc;
	std::map<std::vector<int64_t>, KmPath> pool;
	std::set<std::vector<int64_t>> known;
	int64_t groups = 0;   // shortest_k_groups: the distinct lengths of acc
	bool complete = true; // shortest_k_groups: acc holds every path of the row's first k groups
};

// What a shortest_k_groups call asks of the rounds on top of shortest_k_paths_mode's outputs: k counts length groups,
// max_paths cuts the lists, and the per-row group results (host arrays of p; count nullable)
struct KmGroups {
	int64_t max_paths;
	int64_t *count, *ngroups, *last_len;
	uint8_t *complete;
};

// a spur of the round on the host side: its row and j
struct KmSpurRef {
	int32_t row;
	int32_t j;
};

// the widest lane width of 512 .. 64 whose level array n x W x 2 bytes fits 4 GiB (or opts->lanes)
static int km_lanes_cap(const pgq_options *opts, int64_t n) {
	if (opts && opts->lanes) {
		return opts->lanes;
	}
	int w = 512;
	while (w > 64 && std::max<int64_t>(n, 1) * w * (int64_t)sizeof(uint16_t) > KM_BUDGET) {
		w >>= 1;
	}
	return w;
}

// a round's lane width: the cap, halved while the round's searches are at most half of it (ks_lanes' rule)
static int km_lanes(const pgq_options *opts, const KmSearch &search, int64_t searches) {
	int w = search.cap;
	while (!(opts && opts->lanes) && w > search.lane_min && searches <= w / 2) {
		w >>= 1;
	}
	return w;
}

// shortest_k_paths_mode's spur search: the BFS of the top, level by level over bit masks
struct KmBfs : KmSearch {
	pgq_csr *csr;
	const u64 *step_key = nullptr;
	const int32_t *step_pos = nullptr;
	u64 *seen = nullptr, *front = nullptr, *next = nullptr, *done = nullptr, *grew = nullptr, *ctr = nullptr;
	uint16_t *level = nullptr;
	KmBfs(pgq_csr *c, const pgq_options *opts) : csr(c) {
		cap = km_lanes_cap(opts, c->n);
	}
	int begin(Workspace *ws, const u64 *sk, const int32_t *sp) override {
		const int64_t n = csr->n;
		const int wd_cap = cap / 64;
		step_key = sk;
		step_pos = sp;
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_SEEN, (size_t)n * wd_cap * sizeof(u64), (void **)&seen));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_FRONT, (size_t)n * wd_cap * sizeof(u64), (void **)&front));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_NEXT, (size_t)n * wd_cap * sizeof(u64), (void **)&next));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_LEVEL, (size_t)n * cap * sizeof(uint16_t), (void **)&level));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_DONE, (size_t)wd_cap * sizeof(u64), (void **)&done));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_GREW, (size_t)wd_cap * sizeof(u64), (void **)&grew));
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_COUNTERS, 256, (void **)&ctr));
		return PGQ_OK;
	}
	int has_seed(Workspace *ws, int64_t ns, const KmSpur *spurs, const int32_t *lists, const std::vector<int64_t> &,
	             uint8_t *has, pgq_stats *st) override {
		k_km_has_seed<<<grid_size((ns + 7) / 8, (int64_t)csr->ctx->sm_count * 16), 256, 0, ws->stream>>>(
		    ns, spurs, lists, csr->out.off, csr->out.adj, has);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches++;
		return PGQ_OK;
	}
	int search(Workspace *ws, const KmBatch &b, pgq_stats *st) override {
		cudaStream_t s = ws->stream;
		const int64_t n = csr->n, m = csr->m;
		const int sms = csr->ctx->sm_count;
		const int W = b.W, wd = W / 64, cnt = b.cnt;
		const unsigned edge_grid = grid_size((m + 255) / 256, (int64_t)sms * 16);
		const unsigned vert_grid = grid_size((n + 255) / 256, (int64_t)sms * 8);
		PGQ_CUDA(cudaMemsetAsync(seen, 0, (size_t)n * wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(front, 0, (size_t)n * wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(next, 0, (size_t)n * wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(level, 0xff, (size_t)n * W * sizeof(uint16_t), s));
		PGQ_CUDA(cudaMemsetAsync(done, 0, (size_t)wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(grew, 0, (size_t)wd * sizeof(u64), s));
		PGQ_CUDA(cudaMemsetAsync(b.hlen, 0, (size_t)W * sizeof(int32_t), s));
		PGQ_CUDA(cudaMemsetAsync(ctr, 0, 2 * sizeof(u64), s));
		k_km_seed<<<b.lane_grid, 256, 0, s>>>(cnt, wd, W, b.lane_spur, b.spurs, b.lists, csr->out.off, csr->out.adj,
		                                      seen, front, grew, level, b.ban_bits);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches++;
		for (int lv = 2;; lv++) {
			u64 h_ctr[2];
			PGQ_CUDA(cudaMemsetAsync(&ctr[KM_ACTIVE], 0, sizeof(u64), s));
			k_km_finish<<<1, 1024, 0, s>>>(cnt, wd, W, b.lane_spur, b.spurs, seen, level, grew, done, b.hlen, ctr);
			PGQ_CUDA(cudaGetLastError());
			st->kernel_launches++;
			PGQ_CUDA(cudaMemcpyAsync(h_ctr, ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaMemcpyAsync(b.h_hlen, b.hlen, (size_t)cnt * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st->d2h_bytes += (int64_t)sizeof(h_ctr) + cnt * (int64_t)sizeof(int32_t);
			if (h_ctr[KM_TOO_LONG]) {
				return pgq_fail(PGQ_ERR_UNSUPPORTED, "a spur search went beyond %d edges", KM_PATH_MAX);
			}
			if (!h_ctr[KM_ACTIVE]) {
				break;
			}
			k_km_level<<<edge_grid, 256, 0, s>>>(m, n, wd, csr->out.off, csr->out.adj, front, seen, done, b.ban_bits,
			                                     b.keys, b.nkeys, next);
			k_km_fold<<<vert_grid, 256, 0, s>>>(n, wd, W, lv, seen, front, next, grew, level, ctr);
			PGQ_CUDA(cudaGetLastError());
			st->kernel_launches += 2;
			st->levels++;
		}
		return PGQ_OK;
	}
	int walk(Workspace *ws, const KmBatch &b, const int64_t *lane_off, int2 *steps, longlong2 *step_elems, int64_t *,
	         pgq_stats *st) override {
		k_km_walk<<<b.lane_grid, 256, 0, ws->stream>>>(b.cnt, b.W, csr->n, b.lane_spur, b.spurs, b.lists, b.hlen,
		                                               lane_off, level, csr->in.off, step_key, step_pos, csr->perm,
		                                               csr->inv, csr->out.off, csr->out.adj, csr->edge_ids, steps,
		                                               step_elems);
		PGQ_CUDA(cudaGetLastError());
		st->kernel_launches++;
		return PGQ_OK;
	}
};

int km_run(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
           const uint8_t *dst_valid, const pgq_options *opts, int64_t k, int32_t path_mode, const KmGroups *kg,
           KmSearch &search, int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
           int64_t **out_path_offsets, int64_t **out_elems, void **out_costs, int64_t *out_total_paths,
           pgq_stats *stats) {
	const bool trail = path_mode == PGQ_PATH_TRAIL;
	const bool costs = search.costs;
	const bool f64 = csr->weight_type == 2;
	const int64_t n = csr->n, m = csr->m;
	// c + w in the weight type's arithmetic (a path's sum runs over the edges its search found, below the sentinel)
	auto add = [f64](int64_t c, int64_t w) {
		if (!f64) {
			return c + w;
		}
		double a, b;
		memcpy(&a, &c, sizeof(a));
		memcpy(&b, &w, sizeof(b));
		const double r = a + b;
		int64_t bits;
		memcpy(&bits, &r, sizeof(bits));
		return bits;
	};
	std::vector<int64_t> ids; // the rows whose ids are both valid: sources, then targets
	std::vector<KmRow> rows;
	for (int64_t i = 0; i < p; i++) {
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		if (src[i] < 0 || src[i] >= n || dst[i] < 0 || dst[i] >= n) {
			return pgq_fail(PGQ_ERR_RANGE, "vertex id outside [0, %lld) in row %lld", (long long)n, (long long)i);
		}
		rows.emplace_back();
		rows.back().row = i;
	}
	const int64_t S = (int64_t)rows.size();
	for (const KmRow &r : rows) {
		ids.push_back(src[r.row]);
	}
	for (const KmRow &r : rows) {
		ids.push_back(dst[r.row]);
	}
	const int cap = search.cap;
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	st.lanes = km_lanes(opts, search, 0);
	if (p == 0) {
		PGQ_TRY(empty_lists(out_path_offsets, out_elems, out_costs));
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
	const int sms = csr->ctx->sm_count;
	int32_t *hlen, *pids, *lane_spur;
	int64_t *lane_off;
	uint32_t *ban_bits = nullptr;
	const int64_t *d_ids;
	PGQ_CUDA(cudaEventRecord(ws->ev_begin, s));
	PGQ_TRY(stage_column(ws, WS_KM_IDS, ids.data(), ids.size() * sizeof(int64_t), (const void **)&d_ids));
	st.h2d_bytes += (int64_t)(ids.size() * sizeof(int64_t));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KM_PIDS, ids.size() * sizeof(int32_t), (void **)&pids));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KM_HLEN, (size_t)cap * sizeof(int32_t), (void **)&hlen));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KM_LANE_OFF, (size_t)cap * sizeof(int64_t), (void **)&lane_off));
	PGQ_TRY(pgq_ws_reserve(ws, WS_KM_LANE_SPUR, (size_t)cap * sizeof(int32_t), (void **)&lane_spur));
	if (trail) {
		PGQ_TRY(pgq_ws_reserve(ws, WS_KM_BAN_BITS, (size_t)(m + 31) / 32 * sizeof(uint32_t), (void **)&ban_bits));
	}
	if (S > 0) {
		k_km_ids<<<grid_size((2 * S + 255) / 256, 4096), 256, 0, s>>>(2 * S, d_ids, csr->perm, pids);
		PGQ_CUDA(cudaGetLastError());
		st.kernel_launches++;
	}
	std::vector<int32_t> h_pids(ids.size());
	PGQ_CUDA(cudaMemcpyAsync(h_pids.data(), pids, ids.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	st.d2h_bytes += (int64_t)(ids.size() * sizeof(int32_t));
	for (int64_t i = 0; i < S; i++) {
		rows[i].s = h_pids[i];
		rows[i].t = h_pids[S + i];
	}
	const u64 *step_key = nullptr;
	const int32_t *step_pos = nullptr;
	PGQ_TRY(build_step_lists(csr, ws, s, &step_key, &step_pos, &st.kernel_launches));
	PGQ_TRY(search.begin(ws, step_key, step_pos));
	// ---- rounds ----
	for (int64_t i = 0; i < S; i++) { // s == t: A[0] = [s], no search
		KmRow &r = rows[i];
		if (r.s == r.t) {
			KmPath q;
			q.v.push_back(r.s);
			q.el.push_back(src[r.row]);
			if (costs) {
				q.cost.push_back(0); // (+0 in both weight types)
			}
			r.known.insert(q.key(costs));
			r.acc.push_back(std::move(q));
			r.groups = 1;
			r.live = k > 1;
		}
	}
	for (int64_t round = 0;; round++) {
		std::vector<KmSpur> spurs;
		std::vector<KmSpurRef> refs;
		std::vector<int32_t> lists;
		std::vector<int64_t> roots; // with costs: each spur's root cost
		for (int64_t i = 0; i < S; i++) {
			KmRow &r = rows[i];
			if (!r.live) {
				continue;
			}
			if (round == 0) {
				if (r.s == r.t) {
					continue;
				}
				KmSpur sp = {r.s, r.t, 0, 0, 0, 0, 0, 0, 0};
				spurs.push_back(sp);
				refs.push_back({(int32_t)i, 0});
				roots.push_back(0);
				continue;
			}
			const KmPath &P = r.acc.back();
			const int64_t L = P.h();
			const bool closed = r.s == r.t;
			// TRAIL and WALK spur at j = L too: past t, and back to it
			int64_t j0 = P.dev, j1 = trail || path_mode == PGQ_PATH_WALK ? L : L - 1;
			if (path_mode == PGQ_PATH_SIMPLE && closed && L == 0) {
				j0 = j1 = 0;
			}
			for (int64_t j = j0; j <= j1; j++) {
				KmSpur sp = {P.v[j], r.t, 0, 0, 0, 0, 0, 0, 0};
				sp.vb = (int64_t)lists.size();
				if (path_mode == PGQ_PATH_ACYCLIC || path_mode == PGQ_PATH_SIMPLE) {
					for (int64_t x = 0; x <= j; x++) {
						if (!(closed && P.v[x] == r.t)) {
							lists.push_back(P.v[x]);
						}
					}
				}
				sp.nvb = (int32_t)((int64_t)lists.size() - sp.vb);
				sp.d = (int64_t)lists.size();
				for (const KmPath &Q : r.acc) {
					if (Q.h() > j && std::equal(P.pos.begin(), P.pos.begin() + j, Q.pos.begin())) {
						lists.push_back(Q.pos[j]);
					}
				}
				sp.nd = (int32_t)((int64_t)lists.size() - sp.d);
				sp.eb = (int64_t)lists.size();
				if (trail) {
					lists.insert(lists.end(), P.pos.begin(), P.pos.begin() + j);
				}
				sp.neb = (int32_t)((int64_t)lists.size() - sp.eb);
				spurs.push_back(sp);
				refs.push_back({(int32_t)i, (int32_t)j});
				roots.push_back(costs ? P.cost[j] : 0);
			}
		}
		// the spurs that take a lane
		std::vector<int32_t> lane_of;
		const int64_t ns = (int64_t)spurs.size();
		const KmSpur *d_spurs = nullptr;
		const int32_t *d_lists = nullptr;
		if (ns > 0) {
			uint8_t *d_has;
			PGQ_TRY(stage_column(ws, WS_KM_SPURS, spurs.data(), ns * sizeof(KmSpur), (const void **)&d_spurs));
			PGQ_TRY(stage_column(ws, WS_KM_LISTS, lists.data(), lists.size() * sizeof(int32_t), (const void **)&d_lists));
			if (lists.empty()) {
				PGQ_TRY(pgq_ws_reserve(ws, WS_KM_LISTS, 0, (void **)&d_lists));
			}
			PGQ_TRY(pgq_ws_reserve(ws, WS_KM_HAS_SEED, (size_t)ns, (void **)&d_has));
			PGQ_TRY(search.has_seed(ws, ns, d_spurs, d_lists, roots, d_has, &st));
			std::vector<uint8_t> has((size_t)ns);
			PGQ_CUDA(cudaMemcpyAsync(has.data(), d_has, (size_t)ns, cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaStreamSynchronize(s));
			st.h2d_bytes += (int64_t)(ns * sizeof(KmSpur) + lists.size() * sizeof(int32_t));
			st.d2h_bytes += ns;
			for (int64_t x = 0; x < ns; x++) {
				if (has[x]) {
					lane_of.push_back((int32_t)x);
				}
			}
		}
		const int64_t nl = (int64_t)lane_of.size();
		const int W = km_lanes(opts, search, nl);
		st.lanes = std::max<int32_t>(st.lanes, W);
		st.searches += nl;
		// ---- the round's batches ----
		for (int64_t b0 = 0; b0 < nl; b0 += W) {
			const int cnt = (int)std::min<int64_t>(W, nl - b0);
			const unsigned lane_grid = grid_size((cnt + 7) / 8, (int64_t)sms * 16);
			st.batches++;
			PGQ_CUDA(cudaMemcpyAsync(lane_spur, lane_of.data() + b0, (size_t)cnt * sizeof(int32_t), cudaMemcpyHostToDevice,
			                         s));
			st.h2d_bytes += cnt * (int64_t)sizeof(int32_t);
			// TRAIL: the batch's banned positions as sorted (position, lane) keys
			std::vector<int64_t> keys;
			const int64_t *d_keys = nullptr;
			if (trail) {
				for (int l = 0; l < cnt; l++) {
					const KmSpur &sp = spurs[(size_t)lane_of[(size_t)(b0 + l)]];
					for (int i = 0; i < sp.neb; i++) {
						keys.push_back((int64_t)lists[(size_t)(sp.eb + i)] * 512 + l);
					}
				}
				std::sort(keys.begin(), keys.end());
				if (!keys.empty()) {
					PGQ_CUDA(cudaMemsetAsync(ban_bits, 0, (size_t)(m + 31) / 32 * sizeof(uint32_t), s));
					PGQ_TRY(stage_column(ws, WS_KM_BAN_KEYS, keys.data(), keys.size() * sizeof(int64_t),
					                     (const void **)&d_keys));
					st.h2d_bytes += (int64_t)(keys.size() * sizeof(int64_t));
				}
			}
			std::vector<int32_t> h_hlen((size_t)cnt);
			const KmBatch b = {cnt,       W,      lane_grid, lane_spur, d_spurs, d_lists, d_keys ? ban_bits : nullptr,
			                   d_keys,    (int64_t)keys.size(), hlen, h_hlen.data()};
			PGQ_TRY(search.search(ws, b, &st));
			// ---- walk the found spurs back and add their candidates to the rows' pools ----
			std::vector<int64_t> h_off((size_t)cnt);
			int64_t tot = 0;
			for (int l = 0; l < cnt; l++) {
				h_off[(size_t)l] = tot;
				tot += h_hlen[(size_t)l];
			}
			if (tot == 0) {
				continue;
			}
			int2 *d_steps;
			longlong2 *d_sel;
			int64_t *d_w = nullptr;
			PGQ_TRY(pgq_ws_reserve(ws, WS_KM_STEPS, (size_t)tot * sizeof(int2), (void **)&d_steps));
			PGQ_TRY(pgq_ws_reserve(ws, WS_KM_STEP_ELEMS, (size_t)tot * sizeof(longlong2), (void **)&d_sel));
			if (costs) {
				PGQ_TRY(pgq_ws_reserve(ws, WS_CK_STEP_W, (size_t)tot * sizeof(int64_t), (void **)&d_w));
			}
			PGQ_CUDA(cudaMemcpyAsync(lane_off, h_off.data(), (size_t)cnt * sizeof(int64_t), cudaMemcpyHostToDevice, s));
			PGQ_TRY(search.walk(ws, b, lane_off, d_steps, d_sel, d_w, &st));
			std::vector<int2> h_steps((size_t)tot);
			std::vector<longlong2> h_sel((size_t)tot);
			std::vector<int64_t> h_w(costs ? (size_t)tot : 0);
			PGQ_CUDA(cudaMemcpyAsync(h_steps.data(), d_steps, (size_t)tot * sizeof(int2), cudaMemcpyDeviceToHost, s));
			PGQ_CUDA(cudaMemcpyAsync(h_sel.data(), d_sel, (size_t)tot * sizeof(longlong2), cudaMemcpyDeviceToHost, s));
			if (costs) {
				PGQ_CUDA(cudaMemcpyAsync(h_w.data(), d_w, (size_t)tot * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
				st.d2h_bytes += tot * (int64_t)sizeof(int64_t);
			}
			PGQ_CUDA(cudaStreamSynchronize(s));
			st.h2d_bytes += cnt * (int64_t)sizeof(int64_t);
			st.d2h_bytes += tot * (int64_t)(sizeof(int2) + sizeof(longlong2));
			for (int l = 0; l < cnt; l++) {
				const int64_t h = h_hlen[(size_t)l];
				if (h == 0) {
					continue;
				}
				const KmSpurRef ref = refs[(size_t)lane_of[(size_t)(b0 + l)]];
				KmRow &r = rows[(size_t)ref.row];
				KmPath q;
				q.dev = ref.j;
				if (round == 0) {
					q.v.push_back(r.s);
					q.el.push_back(src[r.row]);
					if (costs) {
						q.cost.push_back(0);
					}
				} else {
					const KmPath &P = r.acc.back();
					q.v.assign(P.v.begin(), P.v.begin() + ref.j + 1);
					q.pos.assign(P.pos.begin(), P.pos.begin() + ref.j);
					q.el.assign(P.el.begin(), P.el.begin() + 2 * ref.j + 1);
					if (costs) {
						q.cost.assign(P.cost.begin(), P.cost.begin() + ref.j + 1);
					}
				}
				for (int64_t i = 0; i < h; i++) {
					const int2 stp = h_steps[(size_t)(h_off[(size_t)l] + i)];
					const longlong2 sel = h_sel[(size_t)(h_off[(size_t)l] + i)];
					const bool last = i == h - 1;
					q.pos.push_back(stp.y);
					q.v.push_back(last ? r.t : h_steps[(size_t)(h_off[(size_t)l] + i + 1)].x);
					q.el.push_back(sel.y);
					q.el.push_back(last ? dst[r.row] : h_sel[(size_t)(h_off[(size_t)l] + i + 1)].x);
					if (costs) {
						q.cost.push_back(add(q.cost.back(), h_w[(size_t)(h_off[(size_t)l] + i)]));
					}
				}
				std::vector<int64_t> key = q.key(costs);
				if (r.known.insert(key).second) {
					r.pool.emplace(std::move(key), std::move(q));
				}
			}
		}
		// ---- each live row accepts its pool's minimum ----
		bool any = false;
		for (KmRow &r : rows) {
			if (!r.live) {
				continue;
			}
			if (round == 0 && r.s == r.t) { // (accepted [s] without a search)
				any = true;
				continue;
			}
			if (r.pool.empty()) {
				r.live = false;
				continue;
			}
			auto it = r.pool.begin();
			if (kg) { // the least path is the row's next: past its k-th group the row is complete, at max_paths cut
				if (r.groups == k && it->second.h() > r.acc.back().h()) {
					r.live = false;
					continue;
				}
				if (kg->max_paths && (int64_t)r.acc.size() == kg->max_paths) {
					r.live = false;
					r.complete = false;
					continue;
				}
			}
			if (it->second.h() > KM_PATH_MAX) {
				return pgq_fail(PGQ_ERR_UNSUPPORTED, "row %lld needs a path longer than %d edges", (long long)r.row,
				                KM_PATH_MAX);
			}
			if (r.acc.empty() || it->second.h() > r.acc.back().h()) {
				r.groups++;
			}
			r.acc.push_back(std::move(it->second));
			r.pool.erase(it);
			r.live = kg || (int64_t)r.acc.size() < k; // (a row of groups spurs off every path it accepts)
			any |= r.live;
		}
		if (!any) {
			break;
		}
	}
	// ---- the rows' lists in pgq_shortest_k_paths' layout ----
	u64 npaths = 0, elem_total = 0;
	for (const KmRow &r : rows) {
		npaths += r.acc.size();
		for (const KmPath &q : r.acc) {
			elem_total += (u64)q.el.size(); // (each path has at most 2 * 65533 + 1 elements)
		}
	}
	if (elem_total > (AS_MAX / sizeof(int64_t)) || npaths > (AS_MAX / sizeof(int64_t)) - 1) {
		return pgq_fail(PGQ_ERR_OOM, "the paths of one call hold too many elements (%llu)", (unsigned long long)elem_total);
	}
	PGQ_CUDA(cudaEventRecord(ws->ev_end, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	g.settled = true;
	float ms = 0.f;
	PGQ_CUDA(cudaEventElapsedTime(&ms, ws->ev_begin, ws->ev_end));
	int64_t *h_off = (int64_t *)malloc((size_t)(npaths + 1) * sizeof(int64_t));
	int64_t *h_elems = (int64_t *)malloc((size_t)std::max<u64>(elem_total, 1) * sizeof(int64_t));
	int64_t *h_costs = out_costs ? (int64_t *)malloc((size_t)std::max<u64>(npaths, 1) * sizeof(int64_t)) : nullptr;
	if (!h_off || !h_elems || (out_costs && !h_costs)) {
		free(h_off);
		free(h_elems);
		free(h_costs);
		return pgq_fail(PGQ_ERR_OOM, "host allocation of %llu path elements failed", (unsigned long long)elem_total);
	}
	memset(out_npaths, 0, (size_t)p * sizeof(int64_t));
	memset(out_valid, 0, (size_t)p);
	for (const KmRow &r : rows) {
		out_npaths[r.row] = (int64_t)r.acc.size();
		out_valid[r.row] = !r.acc.empty();
	}
	if (kg) { // NULL rows: no paths, no groups, complete
		for (int64_t i = 0; i < p; i++) {
			if (kg->count) {
				kg->count[i] = 0;
			}
			kg->ngroups[i] = 0;
			kg->last_len[i] = -1;
			kg->complete[i] = 1;
		}
		for (const KmRow &r : rows) {
			if (kg->count) {
				kg->count[r.row] = r.complete ? (int64_t)r.acc.size() : -1;
			}
			kg->ngroups[r.row] = r.groups;
			kg->last_len[r.row] = r.acc.empty() ? -1 : r.acc.back().h();
			kg->complete[r.row] = r.complete;
		}
	}
	int64_t np = 0, ne = 0;
	size_t ri = 0;
	for (int64_t i = 0; i < p; i++) {
		out_first_path[i] = np;
		if (ri < rows.size() && rows[ri].row == i) {
			for (const KmPath &q : rows[ri].acc) {
				if (h_costs) {
					h_costs[np] = q.cost.back();
				}
				h_off[np++] = ne;
				memcpy(h_elems + ne, q.el.data(), q.el.size() * sizeof(int64_t));
				ne += (int64_t)q.el.size();
			}
			ri++;
		}
	}
	h_off[np] = ne;
	st.total_ms = ms;
	*out_path_offsets = h_off;
	*out_elems = h_elems;
	if (out_costs) {
		*out_costs = h_costs;
	}
	*out_total_paths = np;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_shortest_k_paths_mode(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                         const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                         int64_t k, int32_t path_mode, int64_t *out_npaths, int64_t *out_first_path,
                                         uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
                                         int64_t *out_total_paths, pgq_stats *stats) {
	if (path_mode == PGQ_PATH_WALK) {
		return pgq_shortest_k_paths(csr, p, src, dst, src_valid, dst_valid, opts, k, out_npaths, out_first_path,
		                            out_valid, out_path_offsets, out_elems, out_total_paths, stats);
	}
	if (path_mode != PGQ_PATH_TRAIL && path_mode != PGQ_PATH_ACYCLIC && path_mode != PGQ_PATH_SIMPLE) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "unknown path mode %d", (int)path_mode);
	}
	PGQ_TRY(ks_check_call(csr, p, src, dst, opts, k, out_npaths, out_first_path, out_valid, out_path_offsets, out_elems,
	                      out_total_paths));
	KmBfs bfs(csr, opts);
	return km_run(csr, p, src, dst, src_valid, dst_valid, opts, k, path_mode, nullptr, bfs, out_npaths, out_first_path,
	              out_valid, out_path_offsets, out_elems, nullptr, out_total_paths, stats);
}

extern "C" int pgq_shortest_k_groups(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                     const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                     int64_t k, int32_t path_mode, int64_t max_paths, int64_t *out_count,
                                     int64_t *out_ngroups, int64_t *out_last_len, uint8_t *out_complete,
                                     int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
                                     int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths,
                                     pgq_stats *stats) {
	if (path_mode != PGQ_PATH_WALK && path_mode != PGQ_PATH_TRAIL && path_mode != PGQ_PATH_ACYCLIC &&
	    path_mode != PGQ_PATH_SIMPLE) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "unknown path mode %d", (int)path_mode);
	}
	PGQ_TRY(ks_check_call(csr, p, src, dst, opts, k, out_npaths, out_first_path, out_valid, out_path_offsets, out_elems,
	                      out_total_paths));
	if (p > 0 && (!out_ngroups || !out_last_len || !out_complete)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	if (max_paths < 0) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "max_paths must be >= 0");
	}
	if (path_mode == PGQ_PATH_WALK) {
		return kg_walk(csr, p, src, dst, src_valid, dst_valid, opts, k, max_paths, out_count, out_ngroups, out_last_len,
		               out_complete, out_npaths, out_first_path, out_valid, out_path_offsets, out_elems,
		               out_total_paths, stats);
	}
	const KmGroups kg = {max_paths, out_count, out_ngroups, out_last_len, out_complete};
	KmBfs bfs(csr, opts);
	return km_run(csr, p, src, dst, src_valid, dst_valid, opts, k, path_mode, &kg, bfs, out_npaths, out_first_path,
	              out_valid, out_path_offsets, out_elems, nullptr, out_total_paths, stats);
}
