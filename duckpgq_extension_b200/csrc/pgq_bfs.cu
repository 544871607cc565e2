// pgq_bfs.cu -- multi-source bit-lane BFS on the device CSR: the H100-native replacement of
// IterativeLength / IterativeLengthFunction (reference src/core/functions/scalar/iterativelength.cpp:12-143)
// and of the path variant + ShortestPathFunction (shortest_path.cpp:12-207).  sm_90a only.
//
// State per batch of L = 64*W searches ("lanes"), vertex-major, W x u64 per vertex:
//   seen  [n][W]  lanes that have reached the vertex          (reference: seen)
//   visit [n][W]  lanes whose frontier holds the vertex        (reference: visit)
//   cand  [n][W]  lanes that reach the vertex in this level    (reference: next)
// plus the frontier as a list of work items (vertex, first adjacency position) of <= 1024 edges.
//
// One level is either
//   bottom-up ("pull", dense):  k_pull_fused over the in-edges of every row that can still gain a bit (pgq_pull.cuh:
//       one 32 B-sector gather of the source's visit mask per edge, OR per destination and the level update in the
//       same pass) + k_pull_finish for the rows that cross a range boundary, or
//   top-down ("push", sparse):  k_expand_push over the frontier items only (one warp per item,
//       coalesced adjacency reads, seen-filtered atomicOr into cand) + k_update_sparse over the
//       vertices it touched,
// whose last block also checks which searches reached their destination and publishes the frontier statistics.
// The frontier SETS are identical to the reference's in every level, whichever direction computed
// them, so hop counts, NULLs, the level count and the algorithmic work W are bit-exact.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include <cooperative_groups.h>

#include "pgq_tile.cuh"

namespace cg = cooperative_groups;

#define PGQ_ITEM_EDGES 256 // a frontier work item covers at most this many adjacency positions
#define PGQ_TAIL_MAX 32    // BFS levels one k_tail launch may run
#define PGQ_TAIL_ITEMS 256 // k_tail takes over when the frontier has at most this many items ...
#define PGQ_TAIL_EDGES 1024 // ... and out-edges

template <int W>
struct LaneMask {
	u64 w[W];
};

// device-side level bookkeeping: accumulators written by the update kernels, published (and
// cleared) by the last block of the update kernel (finish_level), then read by the host
struct LevelStatus {
	u64 acc_vertices; // |next frontier|
	u64 acc_edges;    // sum of its out-degrees (= the next level's share of W)
	u64 pub_vertices;
	u64 pub_edges;
	int acc_items; // work items of the next frontier
	int pub_items;
	int n_touched; // vertices first touched by the running push level
	int pub_remaining;
	int err;    // 1 = id out of range
	int total;  // search lanes of this call / shard (k_assign)
	int pruned; // rows answered from the degrees alone (k_assign)
	int search_rows; // rows that are answered by a lane (>= total when sources repeat)
	int batch_n;     // rows attached to the lanes of the running batch (k_init_batch)
	unsigned long long walk_total; // shortestpath: elements of the walked paths so far (slot allocator)
	int tail_levels; // levels run by the last k_tail launch
	int seq;         // host copy only: sequence number of the last publication (see publish_to_host)
	unsigned blocks_done; // ticket counter of the running update kernel (last block finishes the level)
	u64 tail_fv[PGQ_TAIL_MAX]; // |frontier| / out-degree sum produced by each of those levels
	u64 tail_fe[PGQ_TAIL_MAX];
	u64 acc_live[8]; // OR of the new frontier's masks = the lanes whose search is still alive
	u64 pub_live[8];
	u64 acc_gathers; // mask gathers the running bottom-up level really issued (after finished rows)
	u64 pub_gathers;
};

// The host decides the next kernel from the frontier statistics of the finished level.  Instead of a
// D2H copy + stream synchronisation per level, the last thread of a level writes the few numbers
// straight into pinned, device-mapped host memory and then bumps a sequence number the host spins on.
__device__ __forceinline__ void signal_host(LevelStatus *host_st, int seq) {
	__threadfence_system();
	*reinterpret_cast<volatile int *>(&host_st->seq) = seq;
}

// The fields the host reads after every level; the caller then publishes them with signal_host.
__device__ __forceinline__ void publish_fields(LevelStatus *host_st, u64 vertices, u64 edges, int items, int remaining,
                                               u64 gathers, const u64 (&live)[8], int tail_levels) {
	host_st->pub_vertices = vertices;
	host_st->pub_edges = edges;
	host_st->pub_items = items;
	host_st->pub_remaining = remaining;
	host_st->pub_gathers = gathers;
	host_st->tail_levels = tail_levels;
#pragma unroll
	for (int i = 0; i < 8; i++) {
		host_st->pub_live[i] = live[i];
	}
}

// publish_fields from the pub_* fields of the device copy (+ the per-level counts of a k_tail launch)
__device__ __forceinline__ void publish_to_host(LevelStatus *host_st, const LevelStatus *st, int seq, int tail_levels) {
	publish_fields(host_st, st->pub_vertices, st->pub_edges, st->pub_items, st->pub_remaining, st->pub_gathers,
	               st->pub_live, tail_levels);
	for (int i = 0; i < tail_levels; i++) {
		host_st->tail_fv[i] = st->tail_fv[i];
		host_st->tail_fe[i] = st->tail_fe[i];
	}
	signal_host(host_st, seq);
}

// ---- mask loads: one vertex mask = 8*W bytes; W = 4 is exactly one 32 B sector ----------------------
// sm_90 has no 256-bit global access: a 32 B mask is moved as two 128-bit halves (LDG.128 / STG.128) of the
// same sector, issued back to back, so the memory traffic stays one sector per mask.
// PGQ_LD4(Q, p, ...): the 4 x u64 at p (32 B aligned) with the load qualifiers Q (e.g. ".nc.L1::no_allocate").
#define PGQ_LD4(Q, p, m0, m1, m2, m3)                                                                             \
	asm volatile("ld.global" Q ".v2.u64 {%0,%1}, [%4];\n\t"                                                         \
	             "ld.global" Q ".v2.u64 {%2,%3}, [%4+16];"                                                          \
	             : "=&l"(m0), "=&l"(m1), "=&l"(m2), "=&l"(m3) /* early clobber: the address is read after %0 / %1 */  \
	             : "l"(p))

template <int W>
__device__ __forceinline__ void ld_mask(const u64 *__restrict__ base, int64_t idx, u64 (&m)[W]) {
	const u64 *p = base + idx * W;
	if constexpr (W == 1) {
		m[0] = __ldg(p);
	} else if constexpr (W == 2) {
		ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(p));
		m[0] = v.x;
		m[1] = v.y;
	} else {
#pragma unroll
		for (int i = 0; i < W; i += 4) {
			PGQ_LD4(".nc", p + i, m[i], m[i + 1], m[i + 2], m[i + 3]);
		}
	}
}

template <int W>
__device__ __forceinline__ bool any_mask(const u64 (&m)[W]) {
	u64 a = 0;
#pragma unroll
	for (int i = 0; i < W; i++) {
		a |= m[i];
	}
	return a != 0;
}

template <int W>
__device__ __forceinline__ void st_mask(u64 *base, int64_t idx, const u64 (&m)[W]) {
	u64 *p = base + idx * W;
	if constexpr (W == 1) {
		p[0] = m[0];
	} else if constexpr (W == 2) {
		*reinterpret_cast<ulonglong2 *>(p) = make_ulonglong2(m[0], m[1]);
	} else {
#pragma unroll
		for (int i = 0; i < W; i += 4) {
			asm volatile("st.global.v2.u64 [%0], {%1,%2};\n\t"
			             "st.global.v2.u64 [%0+16], {%3,%4};" ::"l"(p + i), "l"(m[i]), "l"(m[i + 1]), "l"(m[i + 2]),
			             "l"(m[i + 3])
			             : "memory");
		}
	}
}

__device__ __forceinline__ u64 warp_or(u64 x) {
	unsigned lo = __reduce_or_sync(FULL_MASK, (unsigned)x);
	unsigned hi = __reduce_or_sync(FULL_MASK, (unsigned)(x >> 32));
	return ((u64)hi << 32) | lo;
}

// ------------------------------------------------------------------------------------------------
// top-down level over the frontier items: for every frontier vertex v and out-edge v -> n:
// cand[n] |= visit[v] & ~seen[n]   (iterativelength.cpp:18-24; the & ~seen filter of l.27 applied
// early, as iterativelength2.cpp:13-31 does).  One warp per item of <= PGQ_ITEM_EDGES edges, four
// 32-edge steps in flight.  The first thread to touch a vertex claims it in tbits; claimed vertices
// are buffered per warp in shared memory and appended to tlist (the next frontier's vertex list)
// with one atomicAdd per ~200 vertices.
// ------------------------------------------------------------------------------------------------
#define PUSH_BUF 256
template <int W, int U, int MB>
__global__ void __launch_bounds__(256, MB) k_expand_push(const int2 *__restrict__ items, int n_items,
                                                     const int32_t *__restrict__ off, const int32_t *__restrict__ adj,
                                                     const u64 *__restrict__ visit, const u64 *__restrict__ seen,
                                                     u64 *__restrict__ cand, uint32_t *tbits, int32_t *tlist,
                                                     LevelStatus *st) {
	__shared__ int32_t buf[8][PUSH_BUF];
	const int lane = threadIdx.x & 31;
	const int wib = threadIdx.x >> 5;
	const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int nwarps = (gridDim.x * blockDim.x) >> 5;
	int buffered = 0; // warp-uniform
	auto flush = [&]() {
		int pos = 0;
		if (lane == 0) {
			pos = atomicAdd(&st->n_touched, buffered);
		}
		pos = __shfl_sync(FULL_MASK, pos, 0);
		__syncwarp();
		for (int i = lane; i < buffered; i += 32) {
			tlist[pos + i] = buf[wib][i];
		}
		__syncwarp();
		buffered = 0;
	};
	for (int it = warp; it < n_items; it += nwarps) {
		const int2 item = items[it];
		const int v = item.x;
		const int end = min(off[v + 1], item.y + PGQ_ITEM_EDGES);
		u64 mv[W];
		ld_mask<W>(visit, v, mv);
		for (int base = item.y; base < end; base += 32 * U) {
			int t[U];
			bool hit[U];
#pragma unroll
			for (int j = 0; j < U; j++) {
				const int e = base + 32 * j + lane;
				t[j] = (e < end) ? adj[e] : -1;
			}
			u64 sn[U][W];
#pragma unroll
			for (int j = 0; j < U; j++) {
				if (t[j] >= 0) {
					ld_mask<W>(seen, t[j], sn[j]);
				}
			}
#pragma unroll
			for (int j = 0; j < U; j++) {
				hit[j] = false;
				if (t[j] >= 0) {
#pragma unroll
					for (int i = 0; i < W; i++) {
						u64 val = mv[i] & ~sn[j][i];
						if (val) {
							atomicOr(&cand[(int64_t)t[j] * W + i], val);
							hit[j] = true;
						}
					}
				}
			}
			uint32_t word[U];
#pragma unroll
			for (int j = 0; j < U; j++) {
				word[j] = hit[j] ? tbits[t[j] >> 5] : 0xffffffffu;
			}
#pragma unroll
			for (int j = 0; j < U; j++) {
				bool is_new = false;
				if (hit[j]) {
					const uint32_t bit = 1u << (t[j] & 31);
					if (!(word[j] & bit)) {
						is_new = !(atomicOr(&tbits[t[j] >> 5], bit) & bit);
					}
				}
				const uint32_t newmask = __ballot_sync(FULL_MASK, is_new);
				if (newmask) {
					if (buffered + 32 > PUSH_BUF) {
						flush();
					}
					if (is_new) {
						buf[wib][buffered + __popc(newmask & (lanemask_le(lane) >> 1))] = t[j];
					}
					buffered += __popc(newmask);
				}
			}
		}
	}
	if (buffered) {
		flush();
	}
}

// Thread-per-item form of the top-down level for frontiers of low-degree vertices (the tail levels
// of a power-law graph hold millions of vertices with a handful of out-edges each): one warp-sized
// group of items is expanded by one warp, every lane walking its own vertex's short adjacency.
template <int W>
__global__ void __launch_bounds__(256) k_expand_push_narrow(const int2 *__restrict__ items, int n_items,
                                                            const int32_t *__restrict__ off,
                                                            const int32_t *__restrict__ adj,
                                                            const u64 *__restrict__ visit, const u64 *__restrict__ seen,
                                                            u64 *__restrict__ cand, uint32_t *tbits, int32_t *tlist,
                                                            LevelStatus *st) {
	const int lane = threadIdx.x & 31;
	for (int it = blockIdx.x * blockDim.x + threadIdx.x; it < n_items; it += gridDim.x * blockDim.x) {
		const int2 item = items[it];
		const int v = item.x;
		const int end = min(off[v + 1], item.y + PGQ_ITEM_EDGES);
		if (item.y >= end) {
			continue;
		}
		u64 mv[W];
		ld_mask<W>(visit, v, mv);
		for (int e = item.y; e < end; e++) {
			const int t = adj[e];
			u64 sn[W];
			ld_mask<W>(seen, t, sn);
			bool hit = false;
#pragma unroll
			for (int i = 0; i < W; i++) {
				u64 val = mv[i] & ~sn[i];
				if (val) {
					atomicOr(&cand[(int64_t)t * W + i], val);
					hit = true;
				}
			}
			bool is_new = false;
			if (hit) {
				const uint32_t bit = 1u << (t & 31);
				if (!(tbits[t >> 5] & bit)) {
					is_new = !(atomicOr(&tbits[t >> 5], bit) & bit);
				}
			}
			const unsigned conv = __activemask();
			const unsigned newmask = __ballot_sync(conv, is_new);
			if (newmask) {
				const int leader = __ffs(newmask) - 1;
				int pos = 0;
				if (lane == leader) {
					pos = atomicAdd(&st->n_touched, __popc(newmask));
				}
				pos = __shfl_sync(conv, pos, leader);
				if (is_new) {
					tlist[pos + __popc(newmask & (lanemask_le(lane) >> 1))] = t;
				}
			}
		}
	}
}

// Appends the work items of a new frontier vertex (warp-aggregated slot reservation).
__device__ __forceinline__ void append_items(bool has, int v, int o0, int o1, int2 *items_next, LevelStatus *st) {
	const int lane = threadIdx.x & 31;
	const int deg = o1 - o0;
	const int mine = has ? max(1, (deg + PGQ_ITEM_EDGES - 1) / PGQ_ITEM_EDGES) : 0;
	int incl = mine;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		int t = __shfl_up_sync(FULL_MASK, incl, d);
		if (lane >= d) {
			incl += t;
		}
	}
	const int total = __shfl_sync(FULL_MASK, incl, 31);
	if (total == 0) {
		return;
	}
	int base = 0;
	if (lane == 31) {
		base = atomicAdd(&st->acc_items, total);
	}
	base = __shfl_sync(FULL_MASK, base, 31) + incl - mine;
	for (int k = 0; k < mine; k++) {
		items_next[base + k] = make_int2(v, o0 + k * PGQ_ITEM_EDGES);
	}
}

template <int W>
__device__ __forceinline__ void record_levels(const u64 (&nx)[W], int64_t v, uint16_t *level, int iter) {
#pragma unroll
	for (int i = 0; i < W; i++) {
		u64 bits = nx[i];
		while (bits) {
			int b = __ffsll((long long)bits) - 1;
			bits &= bits - 1;
			// (a bit is new exactly once; only a source that is re-entered through a cycle gets a second level --
			// k_path_fix_sources puts its 0 back when the batch is over -- so the store needs no read)
			level[v * (int64_t)(64 * W) + 64 * i + b] = (uint16_t)iter;
		}
	}
}

// coherent mask load (no .nc): for data written earlier in the same kernel (k_tail)
template <int W>
__device__ __forceinline__ void ld_mask_coherent(const u64 *base, int64_t idx, u64 (&m)[W]) {
	const volatile u64 *p = base + idx * W;
#pragma unroll
	for (int i = 0; i < W; i++) {
		m[i] = p[i];
	}
}

// Which rows are answered by which search lane (built by k_assign, read-only afterwards, shared by
// all batches of a call).  With one lane per DISTINCT source several rows hang on one lane.
struct LaneMap {
	const int32_t *row_lane; // [p] lane ordinal of the row's search within this call / shard, -1 = none
	const int32_t *lane_src; // [lanes] internal id of the lane's source vertex
	const int32_t *psrc;     // [p] internal vertex ids of the rows
	const int32_t *pdst;
	int64_t p;
};

// What the end of a level needs to see which rows have reached their destination
struct CheckArgs {
	int b0, cnt;               // the running batch = lanes [b0, b0 + cnt)
	const int32_t *batch_rows; // the rows attached to those lanes (LevelStatus::batch_n of them)
	LaneMap lm;
	int64_t *out_len;
	uint8_t *out_valid;
	int iter;
	LevelStatus *host_st;
	int seq;
	int stop_answered; // may the batch end as soon as every row has reached its destination?
};

// ------------------------------------------------------------------------------------------------
// Tail levels in one launch: when the frontier is tiny (the first and the last levels of every
// search, all levels of small or high-diameter graphs) a level costs three launches and a host
// round trip but microseconds of work.  k_tail runs whole levels -- push, update, check -- with ONE
// thread block, block barriers in between, until the frontier dies, every search has finished, the
// frontier outgrows the thresholds, or PGQ_TAIL_MAX levels have run; it records the statistics of
// every level so that the host accounts levels / W exactly as if it had run them one by one.
// ------------------------------------------------------------------------------------------------
template <int W, bool PATH>
__global__ void __launch_bounds__(1024) k_tail(const int32_t *__restrict__ off, const int32_t *__restrict__ adj,
                                               u64 *seen, u64 *buf_visit, u64 *buf_cand, int2 *buf_items,
                                               int2 *buf_items_next, int n_items, int32_t *tlist, uint32_t *tbits,
                                               uint16_t *level, LevelStatus *st, int max_levels, const CheckArgs chk) {
	__shared__ int s_touched, s_items, s_remaining, s_cont;
	__shared__ u64 s_fv, s_fe;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int iter0 = chk.iter;
	const int batch_n = st->batch_n;
	u64 *visit = buf_visit, *cand = buf_cand;
	int2 *items = buf_items, *items_next = buf_items_next;
	int levels = 0;
	for (int lv = 0; lv < max_levels; lv++) {
		if (tid == 0) {
			s_touched = 0;
			s_items = 0;
			s_remaining = 0;
			s_fv = 0;
			s_fe = 0;
		}
		__syncthreads();
		// ---- push: one warp per item
		for (int it = warp; it < n_items; it += 32) {
			const volatile int *ip = reinterpret_cast<const volatile int *>(items + it);
			const int v = ip[0], begin = ip[1];
			const int end = min(off[v + 1], begin + PGQ_ITEM_EDGES);
			u64 mv[W];
			ld_mask_coherent<W>(visit, v, mv);
			for (int e = begin + lane; e < end; e += 32) {
				const int t = adj[e];
				u64 sn[W];
				ld_mask_coherent<W>(seen, t, sn);
				bool hit = false;
#pragma unroll
				for (int i = 0; i < W; i++) {
					u64 val = mv[i] & ~sn[i];
					if (val) {
						atomicOr(&cand[(int64_t)t * W + i], val);
						hit = true;
					}
				}
				if (hit) {
					const uint32_t bit = 1u << (t & 31);
					if (!(atomicOr(&tbits[t >> 5], bit) & bit)) {
						tlist[atomicAdd(&s_touched, 1)] = t;
					}
				}
			}
		}
		__syncthreads();
		// ---- update: new frontier vertices (tlist) + clear the expanded frontier's visit entries
		const int n_touched = s_touched;
		for (int idx = tid; idx < n_touched + n_items; idx += blockDim.x) {
			if (idx < n_touched) {
				const int v = *reinterpret_cast<volatile int32_t *>(tlist + idx);
				u64 nx[W], sn[W];
				ld_mask_coherent<W>(cand, v, nx);
				ld_mask_coherent<W>(seen, v, sn);
#pragma unroll
				for (int i = 0; i < W; i++) {
					sn[i] |= nx[i];
					seen[(int64_t)v * W + i] = sn[i];
				}
				atomicAnd(&tbits[v >> 5], ~(1u << (v & 31)));
				const int o0 = off[v], o1 = off[v + 1];
				atomicAdd(&s_fv, 1ull);
				atomicAdd(&s_fe, (u64)(o1 - o0));
				const int mine = max(1, (o1 - o0 + PGQ_ITEM_EDGES - 1) / PGQ_ITEM_EDGES);
				const int pos = atomicAdd(&s_items, mine);
				for (int k = 0; k < mine; k++) {
					items_next[pos + k] = make_int2(v, o0 + k * PGQ_ITEM_EDGES);
				}
				if (PATH) {
					record_levels<W>(nx, v, level, iter0 + lv);
				}
			} else {
				const int ov = reinterpret_cast<const volatile int *>(items + (idx - n_touched))[0];
#pragma unroll
				for (int i = 0; i < W; i++) {
					visit[(int64_t)ov * W + i] = 0;
				}
			}
		}
		__syncthreads();
		// ---- check: which searches reached their destination (iterativelength.cpp:119-129)
		for (int j = tid; j < batch_n; j += blockDim.x) {
			const int row = chk.batch_rows[j];
			const int l = chk.lm.row_lane[row] - chk.b0;
			const int64_t d = chk.lm.pdst[row];
			const bool found = (*reinterpret_cast<volatile u64 *>(seen + d * W + (l >> 6)) >> (l & 63)) & 1ull;
			if (PATH) {
				if (!found) {
					atomicAdd(&s_remaining, 1);
				}
			} else if (!*reinterpret_cast<volatile uint8_t *>(chk.out_valid + row)) {
				if (found) {
					chk.out_len[row] = iter0 + lv;
					chk.out_valid[row] = 1;
				} else {
					atomicAdd(&s_remaining, 1);
				}
			}
		}
		__syncthreads();
		levels++;
		if (tid == 0) {
			st->tail_fv[lv] = s_fv;
			st->tail_fe[lv] = s_fe;
			const bool finished = chk.stop_answered && s_remaining == 0;
			s_cont = (s_fv > 0 && !finished && s_items <= PGQ_TAIL_ITEMS && s_fe <= PGQ_TAIL_EDGES) ? 1 : 0;
		}
		__syncthreads();
		{ // the frontier just produced becomes the one to expand
			u64 *t = visit;
			visit = cand;
			cand = t;
			int2 *ti = items;
			items = items_next;
			items_next = ti;
		}
		n_items = s_items;
		const int cont = s_cont;
		__syncthreads(); // everybody has read the shared state before the next level resets it
		if (!cont) {
			break;
		}
	}
	if (tid == 0) {
		st->pub_vertices = st->tail_fv[levels - 1];
		st->pub_edges = st->tail_fe[levels - 1];
		st->pub_items = n_items;
		st->pub_remaining = s_remaining;
		st->tail_levels = levels;
		publish_to_host(chk.host_st, st, chk.seq, levels);
	}
}

// ------------------------------------------------------------------------------------------------
// End of a level, run by whichever block of the update kernel finishes last (ticket counter): which
// searches of the batch have reached their destination (iterativelength.cpp:119-129), then publish
// and clear the frontier accumulators.  Saves a kernel launch per level.
// ------------------------------------------------------------------------------------------------
template <int W, bool PATH>
__device__ __forceinline__ void finish_level(LevelStatus *st, const u64 *seen, const CheckArgs &a) {
	__shared__ int s_last, s_remaining;
	__threadfence(); // this block's seen / accumulator updates are visible before its ticket is
	__syncthreads();
	if (threadIdx.x == 0) {
		s_last = (atomicAdd(&st->blocks_done, 1u) == gridDim.x - 1) ? 1 : 0;
		s_remaining = 0;
	}
	__syncthreads();
	if (!s_last) {
		return;
	}
	__threadfence();
	const int batch_n = st->batch_n;
	// R rows per thread and round, their loads issued side by side: one block walks all rows of the batch (up to 1024
	// at 256 threads), and each row is a chain of three dependent loads
	constexpr int R = 4;
	for (int j0 = threadIdx.x; j0 < batch_n; j0 += R * blockDim.x) {
		int row[R];
		bool found[R], answered[R];
#pragma unroll
		for (int r = 0; r < R; r++) {
			const int j = j0 + r * blockDim.x;
			row[r] = j < batch_n ? a.batch_rows[j] : -1;
		}
#pragma unroll
		for (int r = 0; r < R; r++) {
			found[r] = false;
			answered[r] = true;
			if (row[r] >= 0) {
				const int l = a.lm.row_lane[row[r]] - a.b0;
				const int64_t d = a.lm.pdst[row[r]];
				found[r] = (__ldcg(&seen[d * W + (l >> 6)]) >> (l & 63)) & 1ull;
				if (!PATH) {
					answered[r] = *reinterpret_cast<volatile uint8_t *>(a.out_valid + row[r]);
				}
			}
		}
#pragma unroll
		for (int r = 0; r < R; r++) {
			if (row[r] < 0) {
				continue;
			}
			if (PATH) {
				if (!found[r]) {
					atomicAdd(&s_remaining, 1);
				}
			} else if (!answered[r]) {
				if (found[r]) {
					a.out_len[row[r]] = a.iter;
					a.out_valid[row[r]] = 1;
				} else {
					atomicAdd(&s_remaining, 1);
				}
			}
		}
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		// Every block took its ticket behind a fence after its last accumulator update, so L2 loads see the sums.  The
		// loads are issued side by side, and the values go to the host from registers: one atomic read per field, each
		// waiting for the store before it, made this single thread a chain of some twenty memory round trips per level.
		const u64 fv = __ldcg(&st->acc_vertices), fe = __ldcg(&st->acc_edges), gathers = __ldcg(&st->acc_gathers);
		const int items = __ldcg(&st->acc_items);
		u64 live[8];
#pragma unroll
		for (int i = 0; i < 8; i++) {
			live[i] = __ldcg(&st->acc_live[i]);
		}
		st->pub_vertices = fv;
		st->pub_edges = fe;
		st->pub_items = items;
		st->pub_remaining = s_remaining;
		st->pub_gathers = gathers;
#pragma unroll
		for (int i = 0; i < 8; i++) {
			st->pub_live[i] = live[i];
			st->acc_live[i] = 0;
		}
		st->acc_gathers = 0;
		st->acc_vertices = 0;
		st->acc_edges = 0;
		st->acc_items = 0;
		st->n_touched = 0;
		st->blocks_done = 0;
		publish_fields(a.host_st, fv, fe, items, s_remaining, gathers, live, 0);
		signal_host(a.host_st, a.seq);
	}
}

// ------------------------------------------------------------------------------------------------
// update after a push level (iterativelength.cpp:26-30), over the vertices it touched (tlist): seen |= cand; the
// touched vertices are the next frontier (cand becomes its visit array after the host swaps the buffers).  Builds
// the next item list, accumulates |frontier|, its out-degree sum and the live lanes, and, in the same launch, clears
// the visit entries of the frontier that was just expanded.
// mark_seen = 0 is the batch start: the sources enter the frontier WITHOUT being marked seen
// (iterativelength.cpp:86-89,104).
// ------------------------------------------------------------------------------------------------
template <int W, bool PATH>
__global__ void __launch_bounds__(256) k_update_sparse(const int32_t *__restrict__ tlist, const u64 *__restrict__ cand,
                                                       u64 *__restrict__ seen, u64 *__restrict__ old_visit,
                                                       const int2 *__restrict__ old_items, int n_old_items,
                                                       const int32_t *__restrict__ off, uint32_t *tbits,
                                                       int2 *items_next, LevelStatus *st, int mark_seen,
                                                       uint16_t *level, int iter, CheckArgs chk) {
	u64 cnt = 0, edges = 0;
	u64 lv[W];
#pragma unroll
	for (int i = 0; i < W; i++) {
		lv[i] = 0;
	}
	const int n_touched = st->n_touched;
	const int total = n_touched + n_old_items;
	const int nround = (total + 31) & ~31;
	for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < nround; idx += gridDim.x * blockDim.x) {
		bool has = false;
		int v = 0, o0 = 0, o1 = 0;
		if (idx < n_touched) {
			v = tlist[idx];
			u64 nx[W];
			ld_mask<W>(cand, v, nx);
			has = true;
#pragma unroll
			for (int i = 0; i < W; i++) {
				lv[i] |= nx[i];
			}
			if (mark_seen) {
				u64 sn[W];
				ld_mask<W>(seen, v, sn);
#pragma unroll
				for (int i = 0; i < W; i++) {
					sn[i] |= nx[i];
				}
				st_mask<W>(seen, v, sn);
			}
			atomicAnd(&tbits[v >> 5], ~(1u << (v & 31)));
			o0 = off[v];
			o1 = off[v + 1];
			cnt++;
			edges += (u64)(o1 - o0);
			if (PATH && mark_seen) {
				record_levels<W>(nx, v, level, iter);
			}
		} else if (idx < total) {
			const int ov = old_items[idx - n_touched].x;
#pragma unroll
			for (int i = 0; i < W; i++) {
				old_visit[(int64_t)ov * W + i] = 0;
			}
		}
		append_items(has, v, o0, o1, items_next, st);
	}
#pragma unroll
	for (int d = 16; d > 0; d >>= 1) {
		cnt += __shfl_xor_sync(FULL_MASK, cnt, d);
		edges += __shfl_xor_sync(FULL_MASK, edges, d);
	}
	if (cnt) { // (warp-uniform after the reduction)
#pragma unroll
		for (int i = 0; i < W; i++) {
			lv[i] = warp_or(lv[i]);
		}
	}
	if ((threadIdx.x & 31) == 0 && cnt) {
		atomicAdd(&st->acc_vertices, cnt);
		atomicAdd(&st->acc_edges, edges);
#pragma unroll
		for (int i = 0; i < W; i++) {
			if (lv[i]) {
				atomicOr(&st->acc_live[i], lv[i]);
			}
		}
	}
	finish_level<W, PATH>(st, seen, chk);
}

#include "pgq_pull.cuh"

// Behind a fused bottom-up level, one launch (the last block ends the level, finish_level):
//  * The rows that cross a range boundary of k_pull_fused (at most one per range): their OR was combined with
//    atomicOr in cand; apply the level update, and clear them in the array that becomes cand in the next level (a
//    bottom-up level overwrites every exclusive row, so only these must be zero beforehand).  A thread per row; in path
//    mode a warp per row (long rows gain hundreds of bits per level there, which the 32 lanes record together).
//  * Fused bottom-up levels neither gather for nor write finished rows.  A row is marked finished in the level that
//    finds every live lane in its seen mask; the frontier bits it gained in that level (in cand) and in the level
//    before (in visit) are still in the two mask arrays and each must disappear once it has been read as a frontier:
//    when `words` > 0, the rows whose bit appeared in the bitmap since the snapshot taken two levels ago are zeroed in
//    the array that was the level's frontier (old_visit), and the snapshot is refreshed.  (Top-down
//    levels in between clean up after themselves; a stale snapshot only zeroes more rows than necessary, and a finished
//    row's frontier entry may always be zeroed once the level that read it is over.)  A crossing row this launch marks
//    may be missing from the snapshot it writes: its entry in old_visit is cleared by the first part anyway, and a bit
//    missing from a snapshot only makes a later level zero that row once more.
template <int W, bool PATH>
__global__ void __launch_bounds__(256) k_pull_finish(const PullArgs<W> a, u64 *old_visit, uint32_t *snap, int64_t words,
                                                     CheckArgs chk) {
	constexpr int T = PATH ? 32 : 1; // threads per crossing row
	const int lane = threadIdx.x & 31;
	const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
	PullTotals<W> tot;
	for (int64_t i = tid / T; i < a.nranges; i += nthreads / T) {
		const int k = a.shared_row[i]; // rank of a long row
		if (k < 0) {
			continue;
		}
		const int row = a.g.row[k];
		u64 val[W], sn[W];
		ld_mask_rw<W>(a.cand, row, val);
		ld_mask_rw<W>(a.seen, row, sn);
		bool any_new = false, now_sat = true;
#pragma unroll
		for (int w = 0; w < W; w++) {
			val[w] &= ~sn[w];
			any_new |= val[w] != 0;
			sn[w] |= val[w];
			now_sat &= ((~sn[w]) & a.live.w[w]) == 0;
		}
		if (PATH) {
			__syncwarp(); // (all lanes have read the row before lane 0 rewrites it)
		}
		if (!PATH || lane == 0) {
			st_mask<W>(a.cand, row, val);
			if (any_new) {
				st_mask<W>(a.seen, row, sn);
				tot.cnt++;
				tot.edges += (u64)(a.out_off[row + 1] - a.out_off[row]);
#pragma unroll
				for (int w = 0; w < W; w++) {
					tot.live[w] |= val[w];
				}
			}
			if (a.skip && now_sat) {
				atomicOr(&a.satbits[k >> 5], 1u << (k & 31));
			}
#pragma unroll
			for (int w = 0; w < W; w++) {
				old_visit[(int64_t)row * W + w] = 0;
			}
		}
		if (PATH && any_new) {
#pragma unroll
			for (int w = 0; w < W; w++) {
#pragma unroll
				for (int h = 0; h < 2; h++) {
					const int b = lane + 32 * h;
					if ((val[w] >> b) & 1ull) {
						a.level[(int64_t)row * (64 * W) + 64 * w + b] = (uint16_t)a.iter;
					}
				}
			}
		}
	}
	// A warp takes 32 bitmap words, a lane each, then visits only the words with new bits: lane l handles bit l of
	// such a word, so the rank -> row lookups are coalesced.  (Whole warps: nthreads is a multiple of 32.)
	for (int64_t w0 = (tid >> 5) * 32; w0 < words; w0 += nthreads) {
		const int64_t w = w0 + lane;
		uint32_t delta = 0;
		if (w < words) {
			const uint32_t cur = a.satbits[w];
			const uint32_t old = snap[w];
			delta = cur & ~old;
			if (cur != old) {
				snap[w] = cur;
			}
		}
		for (unsigned todo = __ballot_sync(FULL_MASK, delta != 0); todo; todo &= todo - 1) {
			const int j = __ffs(todo) - 1;
			const uint32_t d = __shfl_sync(FULL_MASK, delta, j);
			if ((d >> lane) & 1u) {
				const int64_t idx = (w0 + j) * 32 + lane;
				int row = -1;
				if (idx < a.short_base) {
					if (idx < a.g.n_rows) {
						row = a.g.row[idx];
					}
				} else if (idx - a.short_base < a.g.n_short) {
					row = a.g.s_row[idx - a.short_base];
				}
				if (row >= 0) {
					u64 zero[W];
#pragma unroll
					for (int i = 0; i < W; i++) {
						zero[i] = 0;
					}
					st_mask<W>(old_visit, row, zero);
				}
			}
		}
	}
	pull_totals_flush<W>(tot, a.st);
	finish_level<W, PATH>(a.st, a.seen, chk);
}

// After bottom-up levels the frontier exists only as masks.  When the next level runs top-down (or in
// k_tail) this builds its work-item list and clears the other mask array (which still holds an older
// frontier: fused bottom-up levels do not clean up behind themselves).  Publishes the item count.
template <int W>
__global__ void __launch_bounds__(256) k_frontier_items(int64_t n_rows, const u64 *__restrict__ visit, u64 *other,
                                                        const int32_t *__restrict__ off, int2 *items, LevelStatus *st,
                                                        LevelStatus *host_st, int seq) {
	__shared__ int s_last;
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	const int64_t nround = (n_rows + 31) & ~(int64_t)31; // keep whole warps in the loop (append_items shuffles)
	for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nround; v += stride) {
		bool has = false;
		int o0 = 0, o1 = 0;
		if (v < n_rows) {
			u64 mv[W];
			ld_mask<W>(visit, v, mv);
#pragma unroll
			for (int i = 0; i < W; i++) {
				other[v * W + i] = 0;
			}
			if (any_mask<W>(mv)) {
				has = true;
				o0 = off[v];
				o1 = off[v + 1];
			}
		}
		append_items(has, (int)v, o0, o1, items, st);
	}
	__threadfence();
	__syncthreads();
	if (threadIdx.x == 0) {
		s_last = (atomicAdd(&st->blocks_done, 1u) == gridDim.x - 1) ? 1 : 0;
	}
	__syncthreads();
	if (s_last && threadIdx.x == 0) {
		__threadfence();
		st->pub_items = atomicAdd(&st->acc_items, 0);
		st->acc_items = 0;
		st->blocks_done = 0;
		publish_to_host(host_st, st, seq, 0);
	}
}

// ------------------------------------------------------------------------------------------------
// lane assignment (iterativelength.cpp:93-111 / shortest_path.cpp:106-123).  The reference hands out
// one lane per row in input order; NULL sources (and, for lengths, src == dst) take none.  Here, unless
// the reference's batch composition is asked for (PGQ_OPT_REFERENCE_BATCHING):
//   * rows decided by the degrees alone (source without out-edges, destination without in-edges; for
//     paths also src == dst) are answered on the spot and take no lane (PGQ_OPT_NO_PRUNE switches off);
//   * rows with the SAME source share one lane (PGQ_OPT_NO_DEDUP switches off): the MATCH rewriter
//     emits the cross product of the source and destination sets (match.cpp:476-487), so a chunk of
//     2048 rows often holds a handful of distinct sources.  Lanes are numbered by the first appearance
//     of their source, so without repeated sources this IS the reference's input order.
// With sharding (multi-GPU) a rank keeps the lanes whose ordinal is congruent to its index.
// One cooperative launch, phases separated by grid barriers; every phase is a grid-stride loop over
// the rows in tiles of 1024, so a call with many rows is spread over the SMs.
// ------------------------------------------------------------------------------------------------
struct AssignArgs {
	int64_t p, n;
	const int64_t *src, *dst;
	const uint8_t *src_valid;
	const int32_t *out_off, *in_off, *perm;
	int prune, dedup, shard_index, shard_count;
	int trivial_lanes = 0; // reachability with the reference's batches: src == dst rows search on their source's lane
	int32_t *row_lane, *lane_src, *psrc, *pdst;
	int32_t *row_slot;   // [p] scratch: hash slot of the row's source
	int32_t *hash_key;   // [hash_size] source vertex, -1 = empty
	unsigned *hash_first; // [hash_size] first row with that source
	int32_t *hash_lane;  // [hash_size] lane given to that source
	int hash_size;       // power of two >= 2 p
	int32_t *tile_sum;   // [tiles]
	int32_t *grp_rows;   // [p / 64 + 2] rows attached to each group of 64 lanes
	int64_t *out_len;
	uint8_t *out_valid;
	int64_t *out_lengths; // path mode
	LevelStatus *st;
};

__device__ __forceinline__ unsigned hash_u32(unsigned x) {
	x ^= x >> 16;
	x *= 0x7feb352dU;
	x ^= x >> 15;
	x *= 0x846ca68bU;
	x ^= x >> 16;
	return x;
}

template <bool PATH>
__global__ void __launch_bounds__(1024) k_assign(const AssignArgs a) {
	cg::grid_group grid = cg::this_grid();
	__shared__ int s_warp[32];
	__shared__ int s_base;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + tid, gstride = (int64_t)gridDim.x * blockDim.x;
	const int64_t tiles = (a.p + 1023) / 1024;
	// ---- phase 0: empty hash table / counters
	for (int64_t i = gtid; i < a.hash_size; i += gstride) {
		a.hash_key[i] = -1;
		a.hash_first[i] = 0xffffffffu;
		a.hash_lane[i] = -1;
	}
	for (int64_t i = gtid; i < a.p / 64 + 2; i += gstride) {
		a.grp_rows[i] = 0;
	}
	grid.sync();
	// ---- phase 1: classify the rows; rows that need a search register their source
	int pruned = 0;
	for (int64_t i = gtid; i < a.p; i += gstride) {
		const bool ok = !a.src_valid || a.src_valid[i];
		int slot = -1; // -1: no search, -2: search without de-duplication
		a.out_valid[i] = 0; // NULL / pending
		if (!PATH) {
			a.out_len[i] = -1;
		}
		if (ok) {
			const int64_t sv = a.src[i], dv = a.dst[i];
			if (!PATH && sv == dv && !a.trivial_lanes) {
				a.out_len[i] = 0; // path of length 0 needs no search, iterativelength.cpp:102-103
				a.out_valid[i] = 1;
			} else if (sv < 0 || sv >= a.n || dv < 0 || dv >= a.n) {
				a.st->err = 1;
			} else {
				const int ps = a.perm[sv], pd = a.perm[dv]; // internal ids from here on
				a.psrc[i] = ps;
				a.pdst[i] = pd;
				if (a.prune && PATH && sv == dv) {
					a.out_lengths[i] = -1; // marker: [src], resolved by k_path_offsets
					pruned++;
				} else if (a.prune && sv != dv && (a.out_off[ps + 1] == a.out_off[ps] || a.in_off[pd + 1] == a.in_off[pd])) {
					pruned++; // unreachable: stays NULL
				} else if (!a.dedup) {
					slot = -2;
				} else {
					unsigned h = hash_u32((unsigned)ps) & (unsigned)(a.hash_size - 1);
					for (;;) {
						const int prev = atomicCAS(&a.hash_key[h], -1, ps);
						if (prev == -1 || prev == ps) {
							break;
						}
						h = (h + 1) & (unsigned)(a.hash_size - 1);
					}
					atomicMin(&a.hash_first[h], (unsigned)i);
					slot = (int)h;
				}
			}
		}
		a.row_slot[i] = slot;
		a.row_lane[i] = -1;
	}
	if (pruned) {
		atomicAdd(&a.st->pruned, pruned);
	}
	grid.sync();
	// ---- phase 2: lane leaders (first row of every distinct source) per tile
	for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
		const int64_t i = t * 1024 + tid;
		bool leader = false;
		if (i < a.p) {
			const int slot = a.row_slot[i];
			leader = slot == -2 || (slot >= 0 && a.hash_first[slot] == (unsigned)i);
		}
		const int c = __syncthreads_count(leader);
		if (tid == 0) {
			a.tile_sum[t] = c;
		}
	}
	grid.sync();
	// ---- phase 3: ordinal of every leader in input order -> its lane (this shard's share)
	for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
		int part = 0;
		for (int64_t k = tid; k < t; k += blockDim.x) {
			part += a.tile_sum[k];
		}
#pragma unroll
		for (int d = 16; d > 0; d >>= 1) {
			part += __shfl_xor_sync(FULL_MASK, part, d);
		}
		if (tid == 0) {
			s_base = 0;
		}
		__syncthreads();
		if (lane == 0 && part) {
			atomicAdd(&s_base, part);
		}
		__syncthreads();
		const int64_t i = t * 1024 + tid;
		int slot = -1;
		bool leader = false;
		if (i < a.p) {
			slot = a.row_slot[i];
			leader = slot == -2 || (slot >= 0 && a.hash_first[slot] == (unsigned)i);
		}
		const unsigned bal = __ballot_sync(FULL_MASK, leader);
		if (lane == 0) {
			s_warp[warp] = __popc(bal);
		}
		__syncthreads();
		if (warp == 0) {
			const int w = s_warp[lane];
			int incl = w;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const int x = __shfl_up_sync(FULL_MASK, incl, d);
				if (lane >= d) {
					incl += x;
				}
			}
			s_warp[lane] = incl - w;
		}
		__syncthreads();
		if (leader) {
			const int ord = s_base + s_warp[warp] + __popc(bal & (lanemask_le(lane) >> 1));
			int mine = -1;
			if (a.shard_count <= 1) {
				mine = ord;
			} else if (ord % a.shard_count == a.shard_index) {
				mine = ord / a.shard_count;
			}
			if (mine >= 0) {
				a.lane_src[mine] = a.psrc[i];
			}
			if (slot >= 0) {
				a.hash_lane[slot] = mine;
			} else {
				a.row_lane[i] = mine;
			}
		}
		__syncthreads();
	}
	grid.sync();
	// ---- phase 4: every searching row learns its lane; rows per 64-lane group (sizes the batches' row lists)
	int rows = 0;
	for (int64_t i = gtid; i < a.p; i += gstride) {
		const int slot = a.row_slot[i];
		int l = -1;
		if (slot >= 0) {
			l = a.hash_lane[slot];
			a.row_lane[i] = l;
		} else if (slot == -2) {
			l = a.row_lane[i];
		}
		if (l >= 0) {
			atomicAdd(&a.grp_rows[l >> 6], 1);
			rows++;
		}
	}
	if (rows) {
		atomicAdd(&a.st->search_rows, rows);
	}
	if (gtid == 0) { // lanes of this shard = leaders whose ordinal is congruent to its index
		int all = 0;
		for (int64_t k = 0; k < tiles; k++) {
			all += a.tile_sum[k];
		}
		int minec = all;
		if (a.shard_count > 1) {
			minec = all > a.shard_index ? (all - a.shard_index + a.shard_count - 1) / a.shard_count : 0;
		}
		a.st->total = minec;
	}
}

// Start of a batch: sets the source bits of its lanes in cand (visit1[src][lane] = true,
// iterativelength.cpp:104), lists the distinct source vertices in tlist, and collects the rows that
// are attached to its lanes (batch_rows; LevelStatus::batch_n was zeroed by the host).
template <int W, bool PATH>
__global__ void k_init_batch(int b0, int cnt, LaneMap lm, u64 *cand, uint32_t *tbits, int32_t *tlist, int32_t *batch_rows,
                             LevelStatus *st, uint16_t *level) {
	const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (gtid < cnt) {
		const int l = (int)gtid;
		const int s = lm.lane_src[b0 + l];
		atomicOr(&cand[(int64_t)s * W + (l >> 6)], 1ull << (l & 63));
		const uint32_t bit = 1u << (s & 31);
		if (!(atomicOr(&tbits[s >> 5], bit) & bit)) {
			tlist[atomicAdd(&st->n_touched, 1)] = s;
		}
		if (PATH) {
			level[(int64_t)s * (64 * W) + l] = 0; // parents_v[src][lane] = src, shortest_path.cpp:113-116
		}
	}
	for (int64_t i = gtid; i < lm.p; i += (int64_t)gridDim.x * blockDim.x) {
		const int k = lm.row_lane[i];
		const bool in = k >= b0 && k < b0 + cnt;
		const unsigned bal = __ballot_sync(__activemask(), in);
		if (in) { // warp-aggregated slot reservation
			const int leader = __ffs(bal) - 1;
			int pos = 0;
			if ((threadIdx.x & 31) == leader) {
				pos = atomicAdd(&st->batch_n, __popc(bal));
			}
			pos = __shfl_sync(bal, pos, leader);
			batch_rows[pos + __popc(bal & (lanemask_le(threadIdx.x & 31) >> 1))] = (int32_t)i;
		}
	}
}

// ------------------------------------------------------------------------------------------------
// path reconstruction (shortest_path.cpp:149-204) from the per-(vertex, lane) discovery levels.
// The reference keeps the FIRST parent written while sweeping frontier vertices in ascending id and
// their edges in CSR order (shortest_path.cpp:21-30), i.e. for a node reached at level k:
//   parent = min { v : level[v][lane] == k-1 and v -> node },  edge = first offset of node in adj(parent).
// ------------------------------------------------------------------------------------------------
// blind level stores (record_levels) give a source that is re-entered through a cycle a second level: put the 0 back
// (parents_v[src][lane] = src, shortest_path.cpp:113-116)
__global__ void k_path_fix_sources(int b0, int cnt, int L, const int32_t *__restrict__ lane_src, uint16_t *level) {
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l < cnt) {
		level[(int64_t)lane_src[b0 + l] * L + l] = 0;
	}
}

// per batch: hop count of every row of the batch from the level array (0 = unreachable), and the
// row's slot in the walk buffer (one allocator for the whole call: no host round trip per batch)
__global__ void k_path_batch_lengths(int b0, int L, const int32_t *__restrict__ batch_rows, LaneMap lm,
                                     const uint16_t *__restrict__ level, int64_t *out_lengths, int64_t *slot_off,
                                     LevelStatus *st) {
	const int nb = st->batch_n;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nb; j += gridDim.x * blockDim.x) {
		const int row = batch_rows[j];
		const int l = lm.row_lane[row] - b0;
		const int64_t s = lm.psrc[row], d = lm.pdst[row];
		int64_t len;
		if (s == d) {
			len = 1;
		} else {
			const uint16_t lv = level[d * (int64_t)L + l];
			len = (lv == 0xFFFFu) ? 0 : 2 * (int64_t)lv + 1;
		}
		out_lengths[row] = len;
		slot_off[row] = len > 1 ? (int64_t)atomicAdd(&st->walk_total, (unsigned long long)len) : 0;
	}
}

// whole call, one block: list offsets = exclusive prefix sum of the lengths in row order
// (total_len bookkeeping of shortest_path.cpp:160-203); -1 marks a pruned src == dst row.
__global__ void __launch_bounds__(1024) k_path_offsets(int64_t p, int64_t base, int64_t lo, int64_t hi,
                                                       int64_t *out_offsets, int64_t *out_lengths, uint8_t *out_valid,
                                                       int64_t *range_total) {
	// rows [lo, hi): sequential carry across tiles of 1024 rows
	__shared__ int64_t warp_sums[32];
	__shared__ int64_t carry;
	if (threadIdx.x == 0) {
		carry = base;
	}
	__syncthreads();
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int64_t t0 = lo; t0 < hi; t0 += blockDim.x) {
		int64_t i = t0 + threadIdx.x;
		int64_t len = 0;
		if (i < hi) {
			len = out_lengths[i];
			if (len < 0) {
				len = 1;
				out_lengths[i] = 1;
			}
			out_valid[i] = len > 0;
		}
		int64_t incl = len;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			int64_t t = __shfl_up_sync(FULL_MASK, incl, d);
			if (lane >= d) {
				incl += t;
			}
		}
		if (lane == 31) {
			warp_sums[warp] = incl;
		}
		__syncthreads();
		if (warp == 0) {
			int64_t w = warp_sums[lane];
			int64_t wi = w;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				int64_t t = __shfl_up_sync(FULL_MASK, wi, d);
				if (lane >= d) {
					wi += t;
				}
			}
			warp_sums[lane] = wi - w;
		}
		__syncthreads();
		int64_t excl = carry + warp_sums[warp] + incl - len;
		if (i < hi) {
			out_offsets[i] = excl;
		}
		__syncthreads();
		if (threadIdx.x == blockDim.x - 1) {
			carry = excl + len;
		}
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		*range_total = carry - base;
	}
}

void pgq_path_offsets(int64_t base, int64_t lo, int64_t hi, int64_t *out_offsets, int64_t *out_lengths,
                      uint8_t *out_valid, int64_t *d_range_total, cudaStream_t s) {
	k_path_offsets<<<1, 1024, 0, s>>>(hi, base, lo, hi, out_offsets, out_lengths, out_valid, d_range_total);
}

// [src] lists of the rows that took no lane (pruned src == dst)
__global__ void k_path_trivial(int64_t p, const int64_t *__restrict__ src, const int64_t *__restrict__ dst,
                               const uint8_t *__restrict__ out_valid, const int64_t *__restrict__ out_offsets,
                               const int64_t *__restrict__ out_lengths, int64_t *elems) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p; i += (int64_t)gridDim.x * blockDim.x) {
		if (out_valid[i] && out_lengths[i] == 1) {
			elems[out_offsets[i]] = src[i];
		}
	}
}

// one block per row of the batch (grid-stride): walks back from the destination
__global__ void __launch_bounds__(128) k_path_walk(int b0, int L, const int32_t *__restrict__ batch_rows, LaneMap lm,
                                                   const int64_t *__restrict__ dst, const uint16_t *__restrict__ level,
                                                   DirGraph out, DirGraph in, const int64_t *__restrict__ edge_ids,
                                                   const int32_t *__restrict__ perm, const int32_t *__restrict__ inv,
                                                   const int64_t *__restrict__ slot_off,
                                                   const int64_t *__restrict__ out_lengths, int64_t *walk_elems,
                                                   const LevelStatus *st) {
	__shared__ int best;
	const int nb = st->batch_n;
	for (int j = blockIdx.x; j < nb; j += gridDim.x) {
		const int row = batch_rows[j];
		const int l = lm.row_lane[row] - b0;
		const int64_t len = out_lengths[row];
		if (len <= 1) {
			continue; // unreachable, or [src] (written by k_path_trivial)
		}
		const int64_t off = slot_off[row];
		int cur = lm.pdst[row]; // internal id
		if (threadIdx.x == 0) {
			walk_elems[off + len - 1] = dst[row];
		}
		for (int k = (int)((len - 1) / 2); k >= 1; k--) {
			__syncthreads();
			if (threadIdx.x == 0) {
				best = 0x7fffffff;
			}
			__syncthreads();
			int mine = 0x7fffffff;
			for (int e = in.off[cur] + threadIdx.x; e < in.off[cur + 1]; e += blockDim.x) {
				const int v = in.adj[e];
				if (level[v * (int64_t)L + l] == (uint16_t)(k - 1)) {
					mine = min(mine, inv[v]); // "smallest vertex id" is meant in the ORIGINAL numbering
				}
			}
			if (mine != 0x7fffffff) {
				atomicMin(&best, mine);
			}
			__syncthreads();
			const int parent_orig = best;
			const int parent = perm[parent_orig];
			__syncthreads();
			if (threadIdx.x == 0) {
				best = 0x7fffffff;
			}
			__syncthreads();
			mine = 0x7fffffff;
			for (int e = out.off[parent] + threadIdx.x; e < out.off[parent + 1]; e += blockDim.x) {
				if (out.adj[e] == cur) {
					mine = min(mine, e);
				}
			}
			if (mine != 0x7fffffff) {
				atomicMin(&best, mine);
			}
			__syncthreads();
			const int eoff = best;
			if (threadIdx.x == 0) {
				walk_elems[off + 2 * k - 1] = edge_ids[eoff];
				walk_elems[off + 2 * k - 2] = parent_orig;
			}
			cur = parent;
		}
		__syncthreads();
	}
}

// clears the visit entries of a frontier given as items (used when the batch's very first level is a
// pull level: the sources may lie outside the range the dense update sweeps)
template <int W>
__global__ void k_clear_items(const int2 *__restrict__ items, int n_items, u64 *visit) {
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += gridDim.x * blockDim.x) {
		const int v = items[i].x;
#pragma unroll
		for (int w = 0; w < W; w++) {
			visit[(int64_t)v * W + w] = 0;
		}
	}
}

// after all batches: copy each walked path from its slot in the walk buffer to its final list offset
__global__ void k_path_place(int64_t p, const int32_t *__restrict__ row_lane, const int64_t *__restrict__ slot_off,
                             const int64_t *__restrict__ out_offsets, const int64_t *__restrict__ out_lengths,
                             const int64_t *__restrict__ walk_elems, int64_t *elems) {
	for (int64_t row = blockIdx.x; row < p; row += gridDim.x) {
		if (row_lane[row] < 0) {
			continue;
		}
		const int64_t len = out_lengths[row];
		if (len <= 1) {
			continue;
		}
		const int64_t from = slot_off[row], to = out_offsets[row];
		for (int64_t k = threadIdx.x; k < len; k += blockDim.x) {
			elems[to + k] = walk_elems[from + k];
		}
	}
}

// ------------------------------------------------------------------------------------------------
// host drivers
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// iterativelengthbidirectional (iterativelength_bidirectional.cpp:43-153): every lane runs a search from its source
// (side 0) and one from its destination (side 1), both along out-edges, one side per iteration; the lane is answered
// by the first iteration after which the two seen sets share a vertex.
// ------------------------------------------------------------------------------------------------
// the destination side's seed of every lane (lanes are rows in input order: one row per lane)
__global__ void k_lane_dst(int64_t p, const int32_t *__restrict__ row_lane, const int32_t *__restrict__ pdst,
                           int32_t *lane_dst) {
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p; i += (int64_t)gridDim.x * blockDim.x) {
		const int l = row_lane[i];
		if (l >= 0) {
			lane_dst[l] = pdst[i];
		}
	}
}

// Meet test behind a level of one side (InterSectFronteers, l.34-41, made incremental): seen sets only grow, so the
// intersection after the level is the one before it OR (the level's new bits AND the other side's seen).  The kernel
// walks the new frontier only -- its item list (items != nullptr, LevelStatus::pub_items entries) after a top-down or
// tail level, rows [0, n_rows) after a bottom-up one (a new bit sits on a vertex with an in-edge, and a lane's seeds
// differ, so a meet vertex of a level is never an in-edge-less seed).  The last block answers the rows whose lane met in
// this level with chk.iter, zeroes the accumulator and publishes the rows still open with the level's status.
template <int W>
__global__ void __launch_bounds__(256) k_meet(const u64 *__restrict__ visit, const u64 *__restrict__ other_seen,
                                              const int2 *__restrict__ items, int64_t n_rows, u64 *meet,
                                              const LevelStatus *st, const CheckArgs chk) {
	__shared__ int s_last, s_remaining;
	const int64_t count = items ? (int64_t)st->pub_items : n_rows;
	u64 acc[W];
#pragma unroll
	for (int i = 0; i < W; i++) {
		acc[i] = 0;
	}
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride) {
		const int64_t v = items ? (int64_t)items[k].x : k;
		u64 mv[W], sn[W];
		ld_mask<W>(visit, v, mv);
		ld_mask<W>(other_seen, v, sn);
#pragma unroll
		for (int i = 0; i < W; i++) {
			acc[i] |= mv[i] & sn[i];
		}
	}
#pragma unroll
	for (int i = 0; i < W; i++) {
		acc[i] = warp_or(acc[i]);
		if ((threadIdx.x & 31) == 0 && acc[i]) {
			atomicOr(&meet[i], acc[i]);
		}
	}
	unsigned *ticket = reinterpret_cast<unsigned *>(meet + W);
	__threadfence();
	__syncthreads();
	if (threadIdx.x == 0) {
		s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
		s_remaining = 0;
	}
	__syncthreads();
	if (!s_last) {
		return;
	}
	__threadfence();
	for (int j = threadIdx.x; j < chk.cnt; j += blockDim.x) {
		const int row = chk.batch_rows[j];
		if (chk.out_valid[row]) {
			continue; // met in an earlier iteration
		}
		const int l = chk.lm.row_lane[row] - chk.b0;
		if ((__ldcg(&meet[l >> 6]) >> (l & 63)) & 1ull) {
			chk.out_len[row] = chk.iter;
			chk.out_valid[row] = 1;
		} else {
			atomicAdd(&s_remaining, 1);
		}
	}
	__syncthreads();
	if (threadIdx.x == 0) {
#pragma unroll
		for (int i = 0; i < W; i++) {
			meet[i] = 0;
		}
		*ticket = 0;
		chk.host_st->pub_remaining = s_remaining;
		signal_host(chk.host_st, chk.seq);
	}
}

static inline unsigned grid_cap(int64_t want, int64_t cap) {
	return (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, cap));
}

struct LevelTrace {
	int batch, iter, kind, items; // kind: 0 push, 1 pull, 2 tail (one launch covers several levels)
	int64_t fe, fv;
	int ev; // index of the event pair timing its expansion kernel, -1 = shares the previous one
	int64_t gathers = 0; // bottom-up levels: mask gathers really issued
	int side = -1;       // iterativelengthbidirectional: 0 = the source side, 1 = the destination side
};

// The batches one stream of a call runs, with their counters and level trace
struct Run {
	std::vector<LevelTrace> trace;
	int64_t walk_bound = 0; // shortestpath: upper bound of the walk-buffer elements handed out so far
	pgq_csr *csr;
	Workspace *ws;
	cudaStream_t s;
	pgq_stats st = {};
	size_t ev_used = 0;
	int sms;
	int seq = 0; // sequence number of the last level status the device was asked to publish
	Run(pgq_csr *c, Workspace *w, cudaStream_t stream) : csr(c), ws(w), s(stream), sms(c->ctx->sm_count) {
	}
};

// Adds every additive field of b to a (lanes is the width of a batch, not a count)
static void stats_add(pgq_stats &a, const pgq_stats &b) {
	a.batches += b.batches;
	a.levels += b.levels;
	a.edges_traversed += b.edges_traversed;
	a.frontier_vertices += b.frontier_vertices;
	a.push_levels += b.push_levels;
	a.pull_levels += b.pull_levels;
	a.kernel_launches += b.kernel_launches;
	a.h2d_bytes += b.h2d_bytes;
	a.d2h_bytes += b.d2h_bytes;
	a.expand_ms += b.expand_ms;
	a.total_ms += b.total_ms;
	a.searches += b.searches;
	a.pruned += b.pruned;
	a.search_rows += b.search_rows;
	a.pull_ms += b.pull_ms;
	a.pull_edges += b.pull_edges;
}

// The level status of one stream: a block on the device, zeroed, and the mapped host block it is published into, with
// `extra` bytes behind it
static int status_blocks(Run &r, size_t extra, LevelStatus **d_st, LevelStatus **h_st) {
	PGQ_TRY(pgq_ws_reserve(r.ws, WS_STATUS, sizeof(LevelStatus), (void **)d_st));
	PGQ_TRY(pgq_ws_pinned(r.ws, sizeof(LevelStatus) + extra, (void **)h_st));
	PGQ_CUDA(cudaMemsetAsync(*d_st, 0, sizeof(LevelStatus), r.s));
	return PGQ_OK;
}

// Spins until the device has published status number `seq` into the mapped host block.
static int wait_status(Run &r, LevelStatus *h_st, int seq) {
	volatile int *flag = &h_st->seq;
	for (unsigned spins = 1; *flag != seq; spins++) {
		if ((spins & 0xffff) == 0) {
			std::this_thread::yield(); // a level that takes this long (~ms) need not keep a host core to itself
		}
		if ((spins & 0xfff) == 0) { // every few thousand polls make sure the stream is still healthy
			cudaError_t e = cudaStreamQuery(r.s);
			if (e != cudaSuccess && e != cudaErrorNotReady) {
				cudaGetLastError();
				return pgq_fail(PGQ_ERR_CUDA, "BFS level failed: %s", cudaGetErrorString(e));
			}
			if (e == cudaSuccess && *flag != seq) {
				__sync_synchronize();
				if (*flag != seq) {
					return pgq_fail(PGQ_ERR_CUDA, "BFS level finished without publishing its status");
				}
			}
		}
	}
	__sync_synchronize();
	return PGQ_OK;
}

static int next_event_pair(Run &r, cudaEvent_t *a, cudaEvent_t *b) {
	if (r.ev_used + 2 > r.ws->ev_pool.size()) {
		for (int i = 0; i < 64; i++) {
			cudaEvent_t ev;
			PGQ_CUDA(cudaEventCreate(&ev));
			r.ws->ev_pool.push_back(ev);
		}
	}
	*a = r.ws->ev_pool[r.ev_used];
	*b = r.ws->ev_pool[r.ev_used + 1];
	r.ev_used += 2;
	return PGQ_OK;
}

static int pick_lanes(const pgq_options *opts, int64_t n, int64_t searches, bool path) {
	int lanes = opts ? opts->lanes : 0;
	if (lanes != 0) {
		return lanes;
	}
	// 256 lanes = one 32 B sector per vertex mask: the widest batch whose gather costs a single
	// sector / L1 wavefront per edge.  Narrower when the work on offer is smaller, or when the
	// per-lane level array of the path mode would get too large.
	lanes = 256;
	if (n * 64 <= ((int64_t)32 << 20)) {
		lanes = 512; // small graph: even 64 B masks stay in L2, and half as many batches means half the launches
	}
	if (path) {
		const int64_t budget = (int64_t)4 << 30;
		while (lanes > 64 && n * lanes * 2 > budget) {
			lanes >>= 1;
		}
	}
	while (lanes > 64 && searches <= lanes / 2) {
		lanes >>= 1;
	}
	return lanes;
}

// Everything the batches of one call share (read-only once k_assign has run)
struct CallCtx {
	int64_t p = 0;
	const int64_t *d_src = nullptr, *d_dst = nullptr;
	const pgq_options *opts = nullptr;
	int64_t *d_out_len = nullptr;
	uint8_t *d_out_valid = nullptr;
	int64_t *d_out_lengths = nullptr; // path mode
	int64_t *slot_off = nullptr;      // path mode: [p] slot of a row's walked path in the walk buffer
	PathHook *hook = nullptr;         // path mode: what each batch does instead of shortestpath's walk (nullptr: the walk)
	LaneMap lm;
	const int32_t *h_grp_rows = nullptr; // host copy: rows attached to each group of 64 lanes
	bool ref_batching = false;
	// reachability with the reference's batches (reachability.cpp:15-39,194-235): the sources are seen from the start
	// and a batch runs until a level adds no bit, however many of its rows are answered
	bool reach = false;
	CallCtx(int64_t p_, const int64_t *src, const int64_t *dst, const pgq_options *o, int64_t *out_len,
	        uint8_t *out_valid)
	    : p(p_), d_src(src), d_dst(dst), opts(o), d_out_len(out_len), d_out_valid(out_valid) {
	}
};

// What every level of a batch shares, whichever search side it expands
struct LevelEnv {
	const char *schedule = nullptr; // PGQ_B200_SCHEDULE (see level_env)
	size_t sched_len = 0;
	int direction = 0;
	int64_t alpha = 5;
	int64_t wide_grid = 0;
	bool skip_finished = true;
	bool use_tail = true;
	int64_t n_reach = 0; // only vertices with in-edges can ever enter a frontier after level 0
	unsigned upd_grid = 0;
	int64_t nranges = 0;
	int64_t short_base = 0;
	size_t sat_words = 0; // one finished-rows bitmap; a side owns it and its two snapshots (3 * sat_words)
	int32_t *tlist = nullptr;
	uint32_t *tbits = nullptr;
	int32_t *shared_rows = nullptr;
	uint16_t *level = nullptr;
	LevelStatus *hd_st = nullptr; // device-side address of the mapped host status block
};

// One BFS side of a batch: its mask set, the item lists of its frontier, its finished-rows bitmap (+ snapshots), its
// direction state and what its last level published.  iterativelength runs one side, iterativelengthbidirectional two.
template <int W>
struct BfsSide {
	u64 *seen = nullptr, *visit = nullptr, *cand = nullptr;
	int2 *items = nullptr, *items_next = nullptr;
	uint32_t *satbits = nullptr;
	LaneMask<W> live;        // lanes whose frontier is not empty: only they can still add a bit anywhere
	bool items_valid = true; // does `items` list the current frontier?  (fused bottom-up levels keep only masks)
	int64_t pull_cost = 0;   // gathers the next bottom-up level costs at most: what the last one issued
	int64_t fe = 0, fv = 0;  // the current frontier: out-edges, vertices and work items (as published)
	int n_items = 0;
	int level = 0; // levels this side has run in the batch
	// the frontier statistics the last level published
	void take_status(const LevelStatus *h_st) {
		fe = (int64_t)h_st->pub_edges;
		fv = (int64_t)h_st->pub_vertices;
		n_items = h_st->pub_items;
	}
};

// The per-batch set-up both batch drivers share: the device address of the mapped status block h_st, direction knobs,
// the top-down scratch (tlist / tbits), the bottom-up range scratch and `sides` finished-rows bitmaps with their
// snapshots, the bitmaps zeroed
static int level_env(Run &r, const pgq_options *opts, LevelStatus *h_st, int sides, LevelEnv *e, uint32_t **satbits) {
	pgq_csr *csr = r.csr;
	Workspace *ws = r.ws;
	const int64_t n = csr->n;
	const size_t tbits_bytes = ((size_t)n / 32 + 1) * sizeof(uint32_t);
	PGQ_CUDA(cudaHostGetDevicePointer((void **)&e->hd_st, h_st, 0));
	if (r.seq == 0) {
		*reinterpret_cast<volatile int *>(&h_st->seq) = 0; // forget whatever an earlier call left behind
	}
	PGQ_TRY(pgq_ws_reserve(ws, WS_TLIST, (size_t)std::max<int64_t>(n, 1) * sizeof(int32_t), (void **)&e->tlist));
	PGQ_TRY(pgq_ws_reserve(ws, WS_TBITS, tbits_bytes, (void **)&e->tbits));
	// PGQ_B200_SCHEDULE (tests): the kind of every level, whatever the heuristic would pick.  Character (iter - 1) % len
	// decides level iter (iterativelengthbidirectional: character i % len decides iteration i, of either side):
	// b bottom-up (top-down on an edgeless graph), p top-down, t k_tail where it is eligible (top-down otherwise),
	// a the heuristic.  Overrides opts->direction.
	e->schedule = getenv("PGQ_B200_SCHEDULE");
	e->sched_len = e->schedule ? strlen(e->schedule) : 0;
	if (e->schedule && strspn(e->schedule, "bpta") != e->sched_len) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "PGQ_B200_SCHEDULE may only hold the characters b, p, t and a");
	}
	e->direction = e->sched_len ? 0 : (opts ? opts->direction : 0);
	e->alpha = (opts && opts->alpha > 0) ? opts->alpha : 5; // a pushed edge costs ~5x a pulled one (measured)
	e->wide_grid = (int64_t)r.sms * 8;
	e->skip_finished = !(getenv("PGQ_B200_PULL_SKIP") && atoi(getenv("PGQ_B200_PULL_SKIP")) == 0);
	e->use_tail = !(getenv("PGQ_B200_NO_TAIL") && atoi(getenv("PGQ_B200_NO_TAIL")));
	e->n_reach = csr->n_ab;
	e->upd_grid = grid_cap((e->n_reach + 255) / 256, e->wide_grid);
	e->nranges = (csr->pull.nchunks + PGQ_RANGE_CHUNKS - 1) / PGQ_RANGE_CHUNKS;
	// finished-rows bitmap: the long rows by rank, then (word-aligned) the short rows by sorted position
	e->short_base = (csr->pull.n_rows + 31) / 32 * 32;
	e->sat_words = (size_t)(e->short_base + csr->pull.n_slices * 32) / 32 + 2;
	// (behind the bitmap: its snapshots of one and two levels ago, k_pull_finish)
	const size_t sat_bytes = (size_t)sides * 3 * e->sat_words * sizeof(uint32_t);
	PGQ_TRY(pgq_ws_reserve(ws, WS_SATBITS, sat_bytes, (void **)satbits));
	PGQ_TRY(pgq_ws_reserve(ws, WS_SHARED_ROWS, (size_t)std::max<int64_t>(e->nranges, 1) * sizeof(int32_t),
	                       (void **)&e->shared_rows));
	PGQ_CUDA(cudaMemsetAsync(*satbits, 0, sat_bytes, r.s));
	PGQ_CUDA(cudaMemsetAsync(e->tbits, 0, tbits_bytes, r.s));
	return PGQ_OK;
}

// The workspace slots of a batch's sides (seen, visit, cand, items, items_next): iterativelength runs side 0,
// iterativelengthbidirectional both
static const WsSlot side_slots[2][5] = {{WS_SEEN, WS_VISIT_A, WS_VISIT_B, WS_ITEMS_A, WS_ITEMS_B},
                                        {WS_SEEN_D, WS_VISIT_A_D, WS_VISIT_B_D, WS_ITEMS_A_D, WS_ITEMS_B_D}};

template <int W>
static int reserve_side(Run &r, int k, BfsSide<W> &sd) {
	const int64_t n = r.csr->n;
	const size_t mask_bytes = (size_t)std::max<int64_t>(n, 1) * W * sizeof(u64);
	const size_t items_cap = (size_t)n + (size_t)(r.csr->m / PGQ_ITEM_EDGES) + 64;
	PGQ_TRY(pgq_ws_reserve(r.ws, side_slots[k][0], mask_bytes, (void **)&sd.seen));
	PGQ_TRY(pgq_ws_reserve(r.ws, side_slots[k][1], mask_bytes, (void **)&sd.visit));
	PGQ_TRY(pgq_ws_reserve(r.ws, side_slots[k][2], mask_bytes, (void **)&sd.cand));
	PGQ_TRY(pgq_ws_reserve(r.ws, side_slots[k][3], items_cap * sizeof(int2), (void **)&sd.items));
	PGQ_TRY(pgq_ws_reserve(r.ws, side_slots[k][4], items_cap * sizeof(int2), (void **)&sd.items_next));
	return PGQ_OK;
}

// Level 0 of one side of the batch chk names: k_init_batch lists the batch's rows in batch_rows (= chk.batch_rows) and
// puts the seeds of lane map lm into the side's frontier; k_update_sparse publishes that frontier, marking the seeds
// seen when mark_seen is set.  Rows are answered at level 0 only when `answer` is set: otherwise LevelStatus::batch_n
// is zeroed behind k_init_batch, and the update kernel finds no row to check.
template <int W, bool PATH>
static int seed_side(Run &r, const LevelEnv &env, BfsSide<W> &sd, const LaneMap &lm, bool mark_seen, bool answer,
                     CheckArgs chk, int32_t *batch_rows, LevelStatus *d_st, LevelStatus *h_st) {
	cudaStream_t s = r.s;
	const int cnt = chk.cnt;
	PGQ_CUDA(cudaMemsetAsync(&d_st->batch_n, 0, sizeof(int), s));
	k_init_batch<W, PATH><<<grid_cap((std::max<int64_t>(cnt, lm.p) + 255) / 256, env.wide_grid), 256, 0, s>>>(
	    chk.b0, cnt, lm, sd.cand, env.tbits, env.tlist, batch_rows, d_st, env.level);
	if (!answer) {
		PGQ_CUDA(cudaMemsetAsync(&d_st->batch_n, 0, sizeof(int), s));
	}
	chk.seq = ++r.seq;
	k_update_sparse<W, PATH><<<grid_cap((cnt + 255) / 256, env.wide_grid), 256, 0, s>>>(
	    env.tlist, sd.cand, sd.seen, sd.visit, sd.items, 0, r.csr->out.off, env.tbits, sd.items_next, d_st,
	    mark_seen ? 1 : 0, env.level, 0, chk);
	r.st.kernel_launches += 2;
	PGQ_CUDA(cudaGetLastError());
	std::swap(sd.visit, sd.cand);
	std::swap(sd.items, sd.items_next);
	PGQ_TRY(wait_status(r, h_st, r.seq));
	r.st.d2h_bytes += 64;
	for (int i = 0; i < W; i++) { // the batch's lanes whose frontier is not empty
		const int bits = std::min(64, std::max(0, cnt - 64 * i));
		sd.live.w[i] = (bits >= 64 ? ~0ull : ((1ull << bits) - 1)) & h_st->pub_live[i];
	}
	sd.pull_cost = r.csr->m;
	sd.take_status(h_st);
	return PGQ_OK;
}

// One BFS level of one side: picks its direction (or runs up to max_tail levels in k_tail), launches it, calls
// after_launch(new visit array, new item list or nullptr) -- which may queue more work on the stream and take the
// next status sequence number -- and waits for the level's status.  chk carries everything but the level number and
// sequence number.  *done = levels run (> 1 only for k_tail).  The caller decides from h_st whether the batch goes on.
template <int W, bool PATH, typename AfterLaunch>
static int run_level(Run &r, const LevelEnv &env, BfsSide<W> &sd, LevelStatus *d_st, LevelStatus *h_st, CheckArgs chk,
                     int iter, int64_t sched_pos, int max_tail, AfterLaunch after_launch, int *done) {
	pgq_csr *csr = r.csr;
	cudaStream_t s = r.s;
	const int64_t n = csr->n, m = csr->m;
	const int64_t n_reach = env.n_reach;
	const char forced = env.sched_len ? env.schedule[(size_t)sched_pos % env.sched_len] : 'a';
	const int64_t fe = sd.fe;
	const int64_t fv = sd.fv;
	*done = 1;
	// without an item list its length is bounded by one item per vertex + one per 256 edges
	int n_items = sd.items_valid ? sd.n_items : (int)std::min<int64_t>(fv + fe / PGQ_ITEM_EDGES, 0x7fffffff);
	r.st.levels++;
	r.st.edges_traversed += fe;
	r.st.frontier_vertices += fv;
	// a tiny frontier is expanded by k_tail whatever the direction heuristic says (on a tiny GRAPH
	// every frontier is "large" relative to m, yet three launches + a round trip per level cost
	// far more than the work)
	const bool tail_fits = env.use_tail && n_items <= PGQ_TAIL_ITEMS && fe <= PGQ_TAIL_EDGES;
	bool tail, pull;
	if (forced == 'a') {
		tail = tail_fits && env.direction != 2;
		// (finished rows only ever grow: the gathers of the last bottom-up level bound the next one's)
		pull = !tail && m > 0 && ((env.direction == 2) || (env.direction == 0 && fe * env.alpha > sd.pull_cost));
	} else {
		tail = forced == 't' && tail_fits;
		pull = forced == 'b' && m > 0;
	}
	if (!pull && !sd.items_valid) {
		// top-down after bottom-up: build the frontier's item list from its masks, clean the other array
		k_frontier_items<W><<<env.upd_grid, 256, 0, s>>>(n_reach, sd.visit, sd.cand, csr->out.off, sd.items, d_st,
		                                                 env.hd_st, ++r.seq);
		PGQ_CUDA(cudaGetLastError());
		PGQ_TRY(wait_status(r, h_st, r.seq));
		r.st.kernel_launches++;
		r.st.d2h_bytes += 64;
		n_items = h_st->pub_items;
		sd.items_valid = true;
	}
	r.trace.push_back(LevelTrace {(int)r.st.batches, iter, tail ? 2 : (pull ? 1 : 0), n_items, fe, fv,
	                              (int)(r.ev_used / 2)});
	cudaEvent_t ea, eb;
	PGQ_TRY(next_event_pair(r, &ea, &eb));
	PGQ_CUDA(cudaEventRecord(ea, s));
	chk.iter = iter;
	chk.seq = ++r.seq;
	if (tail) {
		int max_levels = max_tail;
		if (PATH) {
			max_levels = std::min(max_levels, 0xFFFF - iter); // >= 1: no level after 0xFFFE runs (too_deep)
		}
		if (env.sched_len) { // not into a level the schedule gives to b or p
			int run = 1;
			while (run < max_levels && strchr("ta", env.schedule[(size_t)(sched_pos + run) % env.sched_len])) {
				run++;
			}
			max_levels = run;
		}
		k_tail<W, PATH><<<1, 1024, 0, s>>>(csr->out.off, csr->out.adj, sd.seen, sd.visit, sd.cand, sd.items,
		                                  sd.items_next, n_items, env.tlist, env.tbits, env.level, d_st, max_levels, chk);
		PGQ_CUDA(cudaEventRecord(eb, s));
		PGQ_CUDA(cudaGetLastError());
		// (with max_tail == 1 exactly one level runs, and its frontier is in cand / items_next)
		PGQ_TRY(after_launch(sd.cand, sd.items_next));
		PGQ_TRY(wait_status(r, h_st, r.seq));
		r.st.kernel_launches++;
		r.st.d2h_bytes += 64;
		const int ran = h_st->tail_levels;
		r.st.push_levels += ran;
		for (int j = 1; j < ran; j++) { // the levels k_tail ran beyond the first one
			r.st.levels++;
			r.st.edges_traversed += (int64_t)h_st->tail_fe[j - 1];
			r.st.frontier_vertices += (int64_t)h_st->tail_fv[j - 1];
			r.trace.push_back(LevelTrace {(int)r.st.batches, iter + j, 2, -1, (int64_t)h_st->tail_fe[j - 1],
			                              (int64_t)h_st->tail_fv[j - 1], -1});
		}
		if (ran & 1) {
			std::swap(sd.visit, sd.cand);
			std::swap(sd.items, sd.items_next);
		}
		sd.take_status(h_st);
		*done = ran;
		return PGQ_OK;
	}
	if (pull) {
		PullArgs<W> pa;
		pa.g = csr->pull;
		pa.nranges = env.nranges;
		pa.short_base = env.short_base;
		// sources without in-edges hold frontier bits only in the side's first level
		pa.gather_limit = (int32_t)(iter == 1 ? n : n_reach);
		pa.visit = sd.visit;
		pa.seen = sd.seen;
		pa.cand = sd.cand;
		pa.satbits = sd.satbits;
		pa.shared_row = env.shared_rows;
		pa.out_off = csr->out.off;
		pa.st = d_st;
		pa.level = env.level;
		pa.iter = iter;
		pa.skip = env.skip_finished ? 1 : 0;
		pa.live = sd.live;
		// (a warp per range of long rows or slice of short rows)
		const unsigned pull_grid = grid_cap((env.nranges + pa.g.n_slices + 7) / 8, (int64_t)r.sms * PGQ_PULL_CTAS);
		k_pull_fused<W, PATH><<<pull_grid, 256, 0, s>>>(pa);
		PGQ_CUDA(cudaEventRecord(eb, s));
		// (grid-stride loops over a thread per crossing row -- a warp in path mode -- and, when finished rows are
		// skipped, a lane per bitmap word; the snapshot alternates with the level's parity.  Every block takes a
		// ticket of finish_level, so the grid stays at most 8 blocks per SM: on the H100, with a thread per bitmap
		// bit, a cap of 32 blocks per SM ran the bench 4 % slower)
		const int64_t zero_words = env.skip_finished ? (int64_t)env.sat_words : 0;
		const int64_t finish_threads = std::max<int64_t>(env.nranges * (PATH ? 32 : 1), zero_words);
		k_pull_finish<W, PATH><<<grid_cap((finish_threads + 255) / 256, env.wide_grid), 256, 0, s>>>(
		    pa, sd.visit, sd.satbits + env.sat_words * (1 + (iter & 1)), zero_words, chk);
		if (iter == 1) { // the sources may lie outside the rows a bottom-up level rewrites
			k_clear_items<W><<<grid_cap((n_items + 255) / 256, 64), 256, 0, s>>>(sd.items, n_items, sd.visit);
			r.st.kernel_launches++;
		}
		sd.items_valid = false;
		r.st.pull_levels++;
	} else {
		if (fe < (int64_t)n_items * 8) { // low-degree frontier: a thread per item
			k_expand_push_narrow<W><<<grid_cap(((int64_t)n_items + 255) / 256, env.wide_grid), 256, 0, s>>>(
			    sd.items, n_items, csr->out.off, csr->out.adj, sd.visit, sd.seen, sd.cand, env.tbits, env.tlist, d_st);
		} else {
			// (4 x 32 edges in flight, 80 registers; 2 / 1 in flight at higher occupancy measured the same)
			k_expand_push<W, 4, 3><<<grid_cap(((int64_t)n_items + 7) / 8, env.wide_grid), 256, 0, s>>>(
			    sd.items, n_items, csr->out.off, csr->out.adj, sd.visit, sd.seen, sd.cand, env.tbits, env.tlist, d_st);
		}
		PGQ_CUDA(cudaEventRecord(eb, s));
		// grid sized for the worst case the host can bound: every frontier edge touches a new vertex
		const int64_t upper = std::min<int64_t>(fe, n) + n_items;
		k_update_sparse<W, PATH><<<grid_cap((upper + 255) / 256, env.wide_grid), 256, 0, s>>>(
		    env.tlist, sd.cand, sd.seen, sd.visit, sd.items, n_items, csr->out.off, env.tbits, sd.items_next, d_st, 1,
		    env.level, iter, chk);
		r.st.push_levels++;
	}
	r.st.kernel_launches += 2;
	PGQ_CUDA(cudaGetLastError());
	std::swap(sd.visit, sd.cand);
	std::swap(sd.items, sd.items_next);
	PGQ_TRY(after_launch(sd.visit, pull ? nullptr : sd.items));
	PGQ_TRY(wait_status(r, h_st, r.seq));
	r.st.d2h_bytes += 64;
	for (int i = 0; i < W; i++) {
		sd.live.w[i] &= h_st->pub_live[i];
	}
	if (pull) {
		r.trace.back().gathers = (int64_t)h_st->pub_gathers;
		// (+ the walk over the range / slice marks of a level that has nothing left to gather)
		sd.pull_cost = (int64_t)h_st->pub_gathers + m / 256 + 1;
	}
	sd.take_status(h_st);
	return PGQ_OK;
}

template <int W, bool PATH>
static int run_batch(Run &r, const CallCtx &cc, LevelStatus *d_st, LevelStatus *h_st, int b0, int cnt) {
	pgq_csr *csr = r.csr;
	Workspace *ws = r.ws;
	cudaStream_t s = r.s;
	const pgq_options *opts = cc.opts;
	const int64_t n = csr->n, p = cc.p;
	const int L = 64 * W;
	const size_t mask_bytes = (size_t)std::max<int64_t>(n, 1) * W * sizeof(u64);
	BfsSide<W> sd;
	int32_t *batch_rows;
	PGQ_TRY(reserve_side<W>(r, 0, sd));
	PGQ_TRY(pgq_ws_reserve(ws, WS_BATCH_ROWS, (size_t)std::max<int64_t>(p, 1) * sizeof(int32_t), (void **)&batch_rows));
	LevelEnv env;
	if (PATH) {
		PGQ_TRY(pgq_ws_reserve(ws, WS_LEVEL, (size_t)std::max<int64_t>(n, 1) * L * sizeof(uint16_t), (void **)&env.level));
	}
	uint16_t *level = env.level;
	PGQ_TRY(level_env(r, opts, h_st, 1, &env, &sd.satbits));
	const int64_t n_reach = env.n_reach;
	// may the batch end as soon as every row has its destination?  The reference only stops a FULL path
	// batch early (finished_searches == LANE_LIMIT, shortest_path.cpp:144); stopping never changes a path.
	// reachability's batches never stop early (reachability.cpp:205-234)
	const int stop_answered = PATH ? ((!cc.ref_batching || cnt == L) ? 1 : 0) : (cc.reach ? 0 : 1);
	{
		// A batch writes mask rows of vertices with in-edges only (rows < n_reach), except for the source bits of
		// its first level, which that level clears again: once the arrays have been zeroed for this CSR and lane
		// width, later batches clear just the first n_reach rows.
		const bool known = ws->clean_csr_uid == csr->uid && ws->clean_w == W && ws->clean_from == n_reach &&
		                   ws->clean_ptr[0] == sd.seen && ws->clean_ptr[1] == ws->buf[WS_VISIT_A] &&
		                   ws->clean_ptr[2] == ws->buf[WS_VISIT_B];
		const size_t clear_bytes = known ? (size_t)n_reach * W * sizeof(u64) : mask_bytes;
		ws->clean_from = -1; // (until this batch has finished without an error)
		if (clear_bytes > 0) {
			PGQ_CUDA(cudaMemsetAsync(sd.seen, 0, clear_bytes, s));
			PGQ_CUDA(cudaMemsetAsync(sd.visit, 0, clear_bytes, s));
			PGQ_CUDA(cudaMemsetAsync(sd.cand, 0, clear_bytes, s));
		}
	}
	if (PATH) {
		PGQ_CUDA(cudaMemsetAsync(level, 0xFF, (size_t)std::max<int64_t>(n, 1) * L * sizeof(uint16_t), s));
	}
	const CheckArgs chk {b0, cnt, batch_rows, cc.lm, cc.d_out_len, cc.d_out_valid, 0, env.hd_st, 0, stop_answered};
	// (mark_seen: reachability's sources are seen from the start, reachability.cpp:30, iterativelength's are not)
	PGQ_TRY((seed_side<W, PATH>(r, env, sd, cc.lm, cc.reach, true, chk, batch_rows, d_st, h_st)));
	r.st.batches++;
	int iter = 1;
	// Path mode records the level that discovers a vertex in a uint16 array (0xFFFF = unvisited) and supports depths up
	// to 0xFFFD.  A level 0xFFFE still runs: with reference batching a batch ends only at the level that finds its
	// frontier empty, and that level records nothing.  If it finds vertices, the call fails (checked after each level).
	const auto too_deep = [&]() {
		return PATH && iter >= 0xFFFE && h_st->pub_vertices > 0
		           ? pgq_fail(PGQ_ERR_UNSUPPORTED, "BFS deeper than 65533 levels is not supported in path mode")
		           : PGQ_OK;
	};
	const auto no_more = [](const u64 *, const int2 *) { return PGQ_OK; };
	for (;; iter++) {
		int done = 1;
		sd.level = iter;
		PGQ_TRY((run_level<W, PATH>(r, env, sd, d_st, h_st, chk, iter, iter - 1, PGQ_TAIL_MAX, no_more, &done)));
		iter += done - 1;
		PGQ_TRY(too_deep());
		if (h_st->pub_vertices == 0) { // no change, iterativelength.cpp:115-117
			break;
		}
		// every row answered: iterativelength.cpp:114; finished_searches == LANE_LIMIT, shortest_path.cpp:144
		if (stop_answered && h_st->pub_remaining == 0) {
			break;
		}
	}
	if (PATH && cc.hook) {
		int64_t rows_ub = 0;
		for (int g = b0 / 64; g <= (b0 + cnt - 1) / 64; g++) {
			rows_ub += cc.h_grp_rows[g];
		}
		if (rows_ub > 0) {
			k_path_fix_sources<<<(cnt + 127) / 128, 128, 0, s>>>(b0, cnt, L, cc.lm.lane_src, level);
			r.st.kernel_launches++;
			PGQ_CUDA(cudaGetLastError());
			const PathBatch pb {b0, cnt, L, iter, rows_ub, level, batch_rows, &d_st->batch_n, cc.lm.row_lane,
			                    cc.lm.psrc, cc.lm.pdst, cc.d_out_lengths, cc.slot_off, &r.walk_bound, ws, s, &r.st};
			PGQ_TRY(cc.hook->batch(pb));
		}
	} else if (PATH) {
		// Walk this batch's paths into the call's walk buffer (the level array is reused by the next
		// batch).  Slots are handed out on the device; the host only bounds them: a path of this batch
		// has at most 2 * levels + 1 elements, and the rows hanging on its lanes were counted by k_assign.
		int64_t rows_ub = 0;
		for (int g = b0 / 64; g <= (b0 + cnt - 1) / 64; g++) {
			rows_ub += cc.h_grp_rows[g];
		}
		const int64_t bound = rows_ub * (2 * (int64_t)iter + 1);
		int64_t *walk = nullptr;
		PGQ_TRY(pgq_ws_grow(ws, WS_WALK, (size_t)(r.walk_bound + bound) * sizeof(int64_t),
		                    (size_t)r.walk_bound * sizeof(int64_t), s, (void **)&walk));
		r.walk_bound += bound;
		if (rows_ub > 0) {
			k_path_fix_sources<<<(cnt + 127) / 128, 128, 0, s>>>(b0, cnt, L, cc.lm.lane_src, level);
			r.st.kernel_launches++;
			k_path_batch_lengths<<<grid_cap((rows_ub + 127) / 128, env.wide_grid), 128, 0, s>>>(
			    b0, L, batch_rows, cc.lm, level, cc.d_out_lengths, cc.slot_off, d_st);
			k_path_walk<<<grid_cap(rows_ub, (int64_t)r.sms * 16), 128, 0, s>>>(
			    b0, L, batch_rows, cc.lm, cc.d_dst, level, csr->out, csr->in, csr->edge_ids, csr->perm, csr->inv,
			    cc.slot_off, cc.d_out_lengths, walk, d_st);
			r.st.kernel_launches += 2;
			PGQ_CUDA(cudaGetLastError());
		}
	}
	if (cc.reach && n > n_reach) { // seen sources without in-edges: the only rows from n_reach on a batch leaves dirty
		PGQ_CUDA(cudaMemsetAsync(sd.seen + (size_t)n_reach * W, 0, (size_t)(n - n_reach) * W * sizeof(u64), s));
	}
	ws->clean_csr_uid = csr->uid;
	ws->clean_w = W;
	ws->clean_from = n_reach;
	ws->clean_ptr[0] = ws->buf[WS_SEEN];
	ws->clean_ptr[1] = ws->buf[WS_VISIT_A];
	ws->clean_ptr[2] = ws->buf[WS_VISIT_B];
	return PGQ_OK;
}

struct EventGuard { // (error paths must not leak the event)
	cudaEvent_t ev = nullptr;
	~EventGuard() {
		if (ev) {
			cudaEventDestroy(ev);
		}
	}
};

// Start of a call of cc.p > 0 rows: its begin event, the level status (the host block followed by the rows per group of
// 64 lanes) and the lane assignment (k_assign, one cooperative launch), which fills the call's row outputs, cc's lane
// map and the counters of searches, pruned rows and search rows
template <bool PATH>
static int start_call(Run &r, CallCtx &cc, const uint8_t *d_src_valid, int prune, int dedup, int shard_index,
                      int shard_count, LevelStatus **d_st_out, LevelStatus **h_st_out) {
	pgq_csr *csr = r.csr;
	Workspace *ws = r.ws;
	cudaStream_t s = r.s;
	const int64_t p = cc.p;
	PGQ_CUDA(cudaEventRecord(ws->ev_begin, s));
	LevelStatus *d_st, *h_st;
	PGQ_TRY(status_blocks(r, ((size_t)p / 64 + 2) * sizeof(int32_t), &d_st, &h_st));
	*d_st_out = d_st;
	*h_st_out = h_st;
	int32_t *h_grp_rows = reinterpret_cast<int32_t *>(h_st + 1);
	AssignArgs aa;
	aa.trivial_lanes = cc.reach ? 1 : 0;
	aa.p = p;
	aa.n = csr->n;
	aa.src = cc.d_src;
	aa.dst = cc.d_dst;
	aa.src_valid = d_src_valid;
	aa.out_off = csr->out.off;
	aa.in_off = csr->in.off;
	aa.perm = csr->perm;
	aa.prune = prune;
	aa.dedup = dedup;
	aa.shard_index = shard_index;
	aa.shard_count = shard_count;
	int hash_size = 64;
	while ((int64_t)hash_size < 2 * p) {
		hash_size <<= 1;
	}
	aa.hash_size = hash_size;
	const int64_t tiles = (p + 1023) / 1024;
	const size_t tmp_ints = (size_t)p + 3 * (size_t)hash_size + (size_t)tiles + ((size_t)p / 64 + 2);
	int32_t *tmp;
	PGQ_TRY(pgq_ws_reserve(ws, WS_ROW_LANE, (size_t)p * sizeof(int32_t), (void **)&aa.row_lane));
	PGQ_TRY(pgq_ws_reserve(ws, WS_LANE_SRC, (size_t)p * sizeof(int32_t), (void **)&aa.lane_src));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PSRC, (size_t)p * sizeof(int32_t), (void **)&aa.psrc));
	PGQ_TRY(pgq_ws_reserve(ws, WS_PDST, (size_t)p * sizeof(int32_t), (void **)&aa.pdst));
	PGQ_TRY(pgq_ws_reserve(ws, WS_ASSIGN_TMP, tmp_ints * sizeof(int32_t), (void **)&tmp));
	aa.row_slot = tmp;
	aa.hash_key = tmp + p;
	aa.hash_first = reinterpret_cast<unsigned *>(tmp + p + hash_size);
	aa.hash_lane = tmp + p + 2 * (size_t)hash_size;
	aa.tile_sum = tmp + p + 3 * (size_t)hash_size;
	aa.grp_rows = aa.tile_sum + tiles;
	aa.out_len = cc.d_out_len;
	aa.out_valid = cc.d_out_valid;
	aa.out_lengths = cc.d_out_lengths;
	aa.st = d_st;
	{
		void *kargs[] = {(void *)&aa};
		const unsigned grid = grid_cap(tiles, r.sms);
		PGQ_CUDA(cudaLaunchCooperativeKernel((const void *)k_assign<PATH>, dim3(grid), dim3(1024), kargs, 0, s));
	}
	r.st.kernel_launches++;
	PGQ_CUDA(cudaMemcpyAsync(h_st, d_st, sizeof(LevelStatus), cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaMemcpyAsync(h_grp_rows, aa.grp_rows, ((size_t)p / 64 + 2) * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	if (h_st->err) {
		return pgq_fail(PGQ_ERR_RANGE, "source or destination rowid outside [0,%lld)", (long long)csr->n);
	}
	r.st.searches = h_st->total;
	r.st.pruned = h_st->pruned;
	r.st.search_rows = h_st->search_rows;
	cc.lm = LaneMap {aa.row_lane, aa.lane_src, aa.psrc, aa.pdst, p};
	cc.h_grp_rows = h_grp_rows;
	return PGQ_OK;
}

static int check_direction(const pgq_options *opts) {
	if (opts && (opts->direction < 0 || opts->direction > 2)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "direction must be 0, 1 or 2");
	}
	return PGQ_OK;
}

// The reference's batch loop (iterativelength.cpp:84-113, shortest_path.cpp:93-125) starts one batch more when its
// last batch filled every lane (or no row took a lane) and rows that take no lane follow: that batch finds no lane and
// ends at once.  Count it, so that the counters of the reference's batch composition stay the reference's.
static int count_empty_batch(Run &r, const int32_t *row_lane, int64_t p) {
	int32_t last = 0;
	PGQ_CUDA(cudaMemcpyAsync(&last, row_lane + p - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, r.s));
	PGQ_CUDA(cudaStreamSynchronize(r.s));
	if (last < 0) {
		r.st.batches++;
	}
	return PGQ_OK;
}

// The expansion time of a Run's levels (its event pairs), and the time and out-edges of its bottom-up levels, added to
// its stats.  A pair whose time cannot be read is left out; the first such error is returned.
static cudaError_t add_level_times(Run &r, double *expand_ms) {
	const std::vector<cudaEvent_t> &ev = r.ws->ev_pool;
	cudaError_t first = cudaSuccess;
	double acc = 0.0;
	for (size_t i = 0; i + 1 < r.ev_used; i += 2) {
		float t = 0.f;
		const cudaError_t e = cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
		first = first != cudaSuccess ? first : e;
		acc += e == cudaSuccess ? t : 0.f;
	}
	for (const LevelTrace &lt : r.trace) {
		float t = 0.f;
		if (lt.kind == 1 && lt.ev >= 0 && (size_t)(2 * lt.ev + 1) < r.ev_used) {
			const cudaError_t e = cudaEventElapsedTime(&t, ev[2 * lt.ev], ev[2 * lt.ev + 1]);
			first = first != cudaSuccess ? first : e;
			if (e == cudaSuccess) {
				r.st.pull_ms += t;
				r.st.pull_edges += lt.fe;
			}
		}
	}
	r.st.expand_ms += acc;
	*expand_ms = acc;
	return first;
}

// End of a call: its time, the expansion time, the level trace (PGQ_B200_TRACE) and the counters
static int finish_call(Run &r, pgq_stats *stats) {
	Workspace *ws = r.ws;
	cudaStream_t s = r.s;
	PGQ_CUDA(cudaEventRecord(ws->ev_end, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	float ms = 0.f;
	PGQ_CUDA(cudaEventElapsedTime(&ms, ws->ev_begin, ws->ev_end));
	r.st.total_ms = ms;
	double acc = 0.0;
	PGQ_CUDA(add_level_times(r, &acc));
	if (getenv("PGQ_B200_TRACE")) { // development aid: one line per level on stderr
		for (size_t i = 0; i < r.trace.size(); i++) {
			const LevelTrace &lt = r.trace[i];
			float t = 0.f;
			if (lt.ev >= 0 && (size_t)(2 * lt.ev + 1) < r.ev_used) {
				cudaEventElapsedTime(&t, ws->ev_pool[2 * lt.ev], ws->ev_pool[2 * lt.ev + 1]);
			}
			static const char *kinds[3] = {"push", "pull", "tail"};
			if (lt.side >= 0) {
				fprintf(stderr, "[pgq] batch %d iteration %d %s side %s frontier_v=%lld frontier_e=%lld items=%d expand=%.3f ms "
				        "gathers=%lld\n", lt.batch, lt.iter, lt.side ? "dst" : "src", kinds[lt.kind], (long long)lt.fv,
				        (long long)lt.fe, lt.items, t, (long long)lt.gathers);
				continue;
			}
			fprintf(stderr, "[pgq] batch %d level %d %s frontier_v=%lld frontier_e=%lld items=%d expand=%.3f ms gathers=%lld\n",
			        lt.batch, lt.iter, kinds[lt.kind], (long long)lt.fv, (long long)lt.fe, lt.items, t, (long long)lt.gathers);
		}
		fprintf(stderr, "[pgq] call total=%.3f ms expand=%.3f ms lanes=%d searches=%lld rows=%lld pruned=%lld\n",
		        r.st.total_ms, acc, r.st.lanes, (long long)r.st.searches, (long long)r.st.search_rows,
		        (long long)r.st.pruned);
	}
	if (stats) {
		*stats = r.st;
	}
	return PGQ_OK;
}

template <bool PATH>
static int run_call(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                    const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_len, uint8_t *d_out_valid,
                    int64_t *d_out_offsets, int64_t *d_out_lengths, int64_t **d_elems, int64_t *total_out,
                    cudaStream_t s, pgq_stats *stats, bool reach = false, PathHook *hook = nullptr) {
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	if (opts) {
		int l = opts->lanes;
		if (l != 0 && l != 64 && l != 128 && l != 256 && l != 512) {
			return pgq_fail(PGQ_ERR_INVALID_ARG, "lanes must be 0, 64, 128, 256 or 512");
		}
	}
	PGQ_TRY(check_direction(opts));
	Run r(csr, ws, s);
	if (PATH) {
		*d_elems = nullptr;
		*total_out = 0;
	}
	if (p == 0) {
		if (stats) {
			*stats = r.st;
		}
		return PGQ_OK;
	}
	const int flags = opts ? opts->flags : 0;
	const bool ref_batching = (flags & PGQ_OPT_REFERENCE_BATCHING) != 0;
	const int shard_count = (opts && opts->shard_count > 1) ? opts->shard_count : 1;
	const int shard_index = (opts && opts->shard_count > 1) ? opts->shard_index : 0;
	if (shard_index < 0 || shard_index >= shard_count) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "shard_index must lie in [0, shard_count)");
	}
	if (PATH) {
		PGQ_CUDA(cudaMemsetAsync(d_out_offsets, 0, (size_t)p * sizeof(int64_t), s));
		PGQ_CUDA(cudaMemsetAsync(d_out_lengths, 0, (size_t)p * sizeof(int64_t), s));
	}
	CallCtx cc(p, d_src, d_dst, opts, d_out_len, d_out_valid);
	cc.d_out_lengths = d_out_lengths;
	cc.ref_batching = ref_batching;
	cc.reach = reach;
	cc.hook = hook;
	LevelStatus *d_st = nullptr, *h_st = nullptr;
	PGQ_TRY(start_call<PATH>(r, cc, d_src_valid, (ref_batching || (flags & PGQ_OPT_NO_PRUNE)) ? 0 : 1,
	                         (ref_batching || (flags & PGQ_OPT_NO_DEDUP)) ? 0 : 1, shard_index, shard_count, &d_st,
	                         &h_st));
	const int total = h_st->total;
	const int lanes = pick_lanes(opts, csr->n, total, PATH);
	r.st.lanes = lanes;
	if (PATH) {
		PGQ_TRY(pgq_ws_reserve(ws, WS_SLOT_OFF, (size_t)p * sizeof(int64_t), (void **)&cc.slot_off));
	}
	// batches of lanes in assignment order; with lanes = auto the last, partly filled batch uses the
	// narrowest mask that holds it (a 64-lane batch costs about half of a 256-lane one per level)
	struct Batch {
		int pos, take, lanes;
	};
	std::vector<Batch> batches;
	for (int pos = 0; pos < total;) {
		const int remaining = total - pos;
		const int bl = (opts && opts->lanes) ? lanes : pick_lanes(opts, csr->n, remaining, PATH);
		const int take = std::min(remaining, bl);
		batches.push_back(Batch {pos, take, bl});
		pos += take;
	}
	auto run_one = [&](Run &rr, LevelStatus *dst, LevelStatus *hst, const Batch &b) -> int {
		switch (b.lanes) {
#define PGQ_DISPATCH(WW)                                                                                           \
	case 64 * WW:                                                                                                  \
		return run_batch<WW, PATH>(rr, cc, dst, hst, b.pos, b.take);
			PGQ_DISPATCH(1)
			PGQ_DISPATCH(2)
			PGQ_DISPATCH(4)
			PGQ_DISPATCH(8)
#undef PGQ_DISPATCH
		default:
			return pgq_fail(PGQ_ERR_INVALID_ARG, "bad lane width %d", b.lanes);
		}
	};
	// Independent lane batches of one call overlap on an extra stream (own workspace and host thread):
	// while one batch waits for its per-level round trip or runs a light level, another keeps the SMs
	// busy.  Paths stay sequential (they share the level array's workspace and the walk buffer).  The
	// second workspace is only taken if the context's workspace budget allows it.
	int n_streams = getenv("PGQ_B200_BATCH_STREAMS") ? atoi(getenv("PGQ_B200_BATCH_STREAMS")) : 2;
	n_streams = std::max(1, std::min<int>(n_streams, (int)batches.size()));
	std::deque<WsGuard> extra_ws;
	if (!PATH) {
		for (int t = 1; t < n_streams; t++) {
			extra_ws.emplace_back(csr->ctx);
			if (pgq_ws_try_acquire(csr->ctx, &extra_ws.back().ws) != PGQ_OK) {
				extra_ws.pop_back();
				break;
			}
		}
	}
	n_streams = PATH ? 1 : 1 + (int)extra_ws.size();
	// stream t runs batches t, t + n_streams, ...: stream 0 on this thread, every other one on a worker thread
	const auto run_stream = [&](Run &rr, LevelStatus *dst, LevelStatus *hst, int t) -> int {
		int st = PGQ_OK;
		for (size_t i = (size_t)t; i < batches.size() && st == PGQ_OK; i += (size_t)n_streams) {
			st = run_one(rr, dst, hst, batches[i]);
		}
		return st;
	};
	EventGuard assigned; // (the worker streams wait for the lane assignment)
	if (n_streams > 1) {
		cudaError_t ce = cudaEventCreateWithFlags(&assigned.ev, cudaEventDisableTiming);
		if (ce == cudaSuccess) {
			ce = cudaEventRecord(assigned.ev, s);
		}
		if (ce != cudaSuccess) {
			cudaGetLastError();
			return pgq_fail(PGQ_ERR_CUDA, "event setup failed: %s", cudaGetErrorString(ce));
		}
	}
	std::vector<Run> runs; // the workers'
	for (WsGuard &g : extra_ws) {
		runs.emplace_back(csr, g.ws, g.ws->stream);
	}
	std::vector<int> rcs(runs.size(), PGQ_OK);
	std::vector<std::string> errs(runs.size());
	std::vector<std::thread> threads;
	for (size_t t = 0; t < runs.size(); t++) {
		threads.emplace_back([&, t]() {
			Run &rw = runs[t];
			int st = PGQ_OK;
			LevelStatus *dst2 = nullptr, *hst2 = nullptr;
			if (cudaSetDevice(csr->ctx->device) != cudaSuccess ||
			    cudaStreamWaitEvent(rw.s, assigned.ev, 0) != cudaSuccess) {
				st = pgq_fail(PGQ_ERR_CUDA, "worker stream setup failed");
			}
			if (st == PGQ_OK) st = status_blocks(rw, 0, &dst2, &hst2);
			if (st == PGQ_OK) st = run_stream(rw, dst2, hst2, (int)t + 1);
			if (cudaStreamSynchronize(rw.s) != cudaSuccess && st == PGQ_OK) {
				st = pgq_fail(PGQ_ERR_CUDA, "worker stream failed");
			}
			if (st != PGQ_OK) {
				errs[t] = pgq_last_error(); // thread-local message of this worker
			}
			rcs[t] = st;
		});
	}
	int rc = run_stream(r, d_st, h_st, 0);
	for (auto &th : threads) {
		th.join();
	}
	for (WsGuard &g : extra_ws) {
		g.settled = true; // (its worker has waited for its stream)
	}
	for (size_t t = 0; t < runs.size(); t++) { // fold the workers' counters and level times into the call's
		double expand_ms;
		(void)add_level_times(runs[t], &expand_ms); // (a failed worker may leave a pair unrecorded: it is left out)
		stats_add(r.st, runs[t].st);
		if (rc == PGQ_OK && rcs[t] != PGQ_OK) {
			rc = pgq_fail(rcs[t], "%s", errs[t].c_str());
		}
	}
	extra_ws.clear(); // (back to the pool)
	if (rc != PGQ_OK) {
		return rc;
	}
	// (Only at an explicit lane width: with lanes = auto the last batch is narrowed to what it holds, so "full" says
	// nothing about the reference's batches.)
	if (ref_batching && opts && opts->lanes && p > 0 && shard_count <= 1 &&
	    (batches.empty() || batches.back().take == batches.back().lanes)) {
		PGQ_TRY(count_empty_batch(r, cc.lm.row_lane, p));
	}
	if (PATH && (!hook || hook->lists)) {
		// list offsets over ALL rows in row order, then move every walked path to its place
		int64_t *d_total;
		PGQ_TRY(pgq_ws_reserve(ws, WS_PATH_TOTAL, 256, (void **)&d_total));
		k_path_offsets<<<1, 1024, 0, s>>>(p, 0, 0, p, d_out_offsets, d_out_lengths, d_out_valid, d_total);
		int64_t list_total = 0;
		PGQ_CUDA(cudaMemcpyAsync(&list_total, d_total, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaStreamSynchronize(s));
		int64_t *elems = nullptr;
		PGQ_TRY(pgq_ws_reserve(ws, WS_ELEMS, (size_t)std::max<int64_t>(list_total, 1) * sizeof(int64_t), (void **)&elems));
		k_path_trivial<<<grid_cap((p + 255) / 256, 1024), 256, 0, s>>>(p, d_src, d_dst, d_out_valid, d_out_offsets,
		                                                              d_out_lengths, elems);
		if (total > 0 && r.walk_bound > 0) {
			k_path_place<<<grid_cap(p, 4096), 64, 0, s>>>(p, cc.lm.row_lane, cc.slot_off, d_out_offsets, d_out_lengths,
			                                             (const int64_t *)ws->buf[WS_WALK], elems);
		}
		r.st.kernel_launches += 3;
		PGQ_CUDA(cudaGetLastError());
		*d_elems = elems; // lives in the workspace: valid until the caller releases it
		*total_out = list_total;
	}
	return finish_call(r, stats);
}

int pgq_bfs_lengths_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                           const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_len,
                           uint8_t *d_out_valid, cudaStream_t stream, pgq_stats *stats) {
	return run_call<false>(csr, ws, p, d_src, d_dst, d_src_valid, opts, d_out_len, d_out_valid, nullptr, nullptr,
	                       nullptr, nullptr, stream, stats);
}

int pgq_bfs_paths_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                         const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_offsets,
                         int64_t *d_out_lengths, uint8_t *d_out_valid, int64_t **d_out_elems, int64_t *out_total,
                         cudaStream_t stream, pgq_stats *stats) {
	return run_call<true>(csr, ws, p, d_src, d_dst, d_src_valid, opts, nullptr, d_out_valid, d_out_offsets,
	                      d_out_lengths, d_out_elems, out_total, stream, stats);
}

int pgq_bfs_paths_hooked(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                         const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_offsets,
                         int64_t *d_out_lengths, uint8_t *d_out_valid, int64_t **d_out_elems, int64_t *out_total,
                         PathHook *hook, cudaStream_t stream, pgq_stats *stats) {
	return run_call<true>(csr, ws, p, d_src, d_dst, d_src_valid, opts, nullptr, d_out_valid, d_out_offsets,
	                      d_out_lengths, d_out_elems, out_total, stream, stats, false, hook);
}

// reachability (reachability.cpp:165-254): row i is true when its search finds dst[i] (d_out_valid[i] = 1).
// By default the rows run exactly as pgq_iterativelength runs them.  With PGQ_OPT_REFERENCE_BATCHING the rows are cut
// into the reference's batches on the host (InitialiseBfs, l.15-39): in input order, a row whose source is new to the
// batch opens the next lane, a row whose source is not shares its lane (src == dst rows too), a NULL source takes
// none, and the batch ends behind the row that opened lane 512.  Unlike the reference's restart (l.251, which counts
// the valid rows only), NULL sources do not move the next batch's start.  Each batch is one run_call of its rows at 512
// lanes, de-duplication on and the degree shortcut off, in reachability's mode (CallCtx::reach).
int pgq_bfs_reachability_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                                const uint8_t *d_src_valid, const int64_t *h_src, const uint8_t *h_src_valid,
                                const pgq_options *opts, int64_t *d_out_len, uint8_t *d_out_valid, cudaStream_t s,
                                pgq_stats *stats) {
	if (opts && opts->shard_count > 1) {
		return pgq_fail(PGQ_ERR_UNSUPPORTED, "reachability takes no sharding");
	}
	if (!opts || !(opts->flags & PGQ_OPT_REFERENCE_BATCHING)) {
		return run_call<false>(csr, ws, p, d_src, d_dst, d_src_valid, opts, d_out_len, d_out_valid, nullptr, nullptr,
		                       nullptr, nullptr, s, stats);
	}
	if (opts->lanes != 0 && opts->lanes != 512) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "reachability's reference batches have 512 lanes: lanes must be 0 or 512");
	}
	constexpr int L = 512; // LANE_LIMIT
	pgq_options bo = *opts;
	bo.lanes = L;
	bo.flags = PGQ_OPT_NO_PRUNE;
	bo.shard_index = 0;
	bo.shard_count = 0;
	pgq_stats sum;
	memset(&sum, 0, sizeof(sum));
	sum.lanes = L;
	std::unordered_set<int64_t> lanes;
	lanes.reserve(2 * L);
	for (int64_t b0 = 0; b0 < p;) {
		int64_t end = b0;
		lanes.clear();
		for (; end < p && lanes.size() < (size_t)L; end++) {
			if (!h_src_valid || h_src_valid[end]) {
				lanes.insert(h_src[end]);
			}
		}
		pgq_stats st;
		PGQ_TRY(run_call<false>(csr, ws, end - b0, d_src + b0, d_dst + b0, d_src_valid ? d_src_valid + b0 : nullptr, &bo,
		                        d_out_len + b0, d_out_valid + b0, nullptr, nullptr, nullptr, nullptr, s, &st, true));
		stats_add(sum, st);
		b0 = end;
	}
	if (stats) {
		*stats = sum;
	}
	return PGQ_OK;
}

// One batch of iterativelengthbidirectional (l.84-151) at L = 64 * W lanes [b0, b0 + cnt): both sides are seeded (their
// seeds seen from the start, l.107-110), then iteration i runs one level of side i & 1 through run_level -- the same
// level kernels and direction choice as iterativelength, each side with its own direction state -- followed by
// k_meet.  The update kernels answer no row here (LevelStatus::batch_n stays 0); k_meet does.  A met lane keeps
// expanding: its bits decide, with everybody else's, whether the batch goes on (l.119-128).
template <int W>
static int run_bidir_batch(Run &r, const CallCtx &cc, const LaneMap &lm_dst, LevelStatus *d_st, LevelStatus *h_st,
                           int b0, int cnt) {
	pgq_csr *csr = r.csr;
	Workspace *ws = r.ws;
	cudaStream_t s = r.s;
	const int64_t n = csr->n, p = cc.p;
	const size_t mask_bytes = (size_t)std::max<int64_t>(n, 1) * W * sizeof(u64);
	BfsSide<W> side[2];
	for (int k = 0; k < 2; k++) {
		PGQ_TRY(reserve_side<W>(r, k, side[k]));
	}
	int32_t *batch_rows;
	u64 *meet;
	PGQ_TRY(pgq_ws_reserve(ws, WS_BATCH_ROWS, (size_t)std::max<int64_t>(p, 1) * sizeof(int32_t), (void **)&batch_rows));
	PGQ_TRY(pgq_ws_reserve(ws, WS_MEET, (W + 1) * sizeof(u64), (void **)&meet));
	LevelEnv env;
	uint32_t *satbits = nullptr;
	PGQ_TRY(level_env(r, cc.opts, h_st, 2, &env, &satbits));
	side[0].satbits = satbits;
	side[1].satbits = satbits + 3 * env.sat_words;
	// Seeds stay seen, so rows beyond n_reach get written: the known-zero rows of the search slots are not kept up here,
	// and both mask sets are cleared whole.
	ws->clean_from = -1;
	PGQ_CUDA(cudaMemsetAsync(meet, 0, (W + 1) * sizeof(u64), s));
	for (int k = 0; k < 2; k++) {
		PGQ_CUDA(cudaMemsetAsync(side[k].seen, 0, mask_bytes, s));
		PGQ_CUDA(cudaMemsetAsync(side[k].visit, 0, mask_bytes, s));
		PGQ_CUDA(cudaMemsetAsync(side[k].cand, 0, mask_bytes, s));
	}
	// no row is answered by the update kernels, k_meet answers them: each k_init_batch lists the batch's rows, one per
	// lane, in batch_rows, and the seeds are seen from the start
	const CheckArgs chk {b0, cnt, batch_rows, cc.lm, cc.d_out_len, cc.d_out_valid, 0, env.hd_st, 0, 0};
	for (int k = 0; k < 2; k++) {
		PGQ_TRY((seed_side<W, false>(r, env, side[k], k ? lm_dst : cc.lm, true, false, chk, batch_rows, d_st,
		                                    h_st)));
	}
	r.st.batches++;
	for (int it = 0;; it++) {
		BfsSide<W> &sd = side[it & 1];
		const u64 *other_seen = side[(it & 1) ^ 1].seen;
		const auto meet_test = [&](const u64 *new_visit, const int2 *new_items) -> int {
			CheckArgs mc = chk;
			mc.iter = it + 1; // found at iteration it => length it + 1 (l.135)
			mc.seq = ++r.seq;
			k_meet<W><<<env.upd_grid, 256, 0, s>>>(new_visit, other_seen, new_items, env.n_reach, meet, d_st, mc);
			r.st.kernel_launches++;
			PGQ_CUDA(cudaGetLastError());
			return PGQ_OK;
		};
		int done = 1;
		sd.level++;
		PGQ_TRY((run_level<W, false>(r, env, sd, d_st, h_st, chk, sd.level, it, 1, meet_test, &done)));
		r.trace.back().iter = it;
		r.trace.back().side = it & 1;
		if (h_st->pub_vertices == 0) { // no lane of the batch gained a bit on this side, l.120-127
			break;
		}
		if (h_st->pub_remaining == 0) { // every lane has met
			break;
		}
	}
	return PGQ_OK;
}

int pgq_bfs_bidirectional_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                                 const uint8_t *d_valid, const pgq_options *opts, int64_t *d_out_len,
                                 uint8_t *d_out_valid, cudaStream_t s, pgq_stats *stats) {
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	if (opts && opts->lanes != 0 && opts->lanes != 512) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "iterativelengthbidirectional runs 512 lanes per batch: lanes must be 0 or 512");
	}
	PGQ_TRY(check_direction(opts));
	if (opts && (opts->flags != 0 || opts->shard_count > 1)) {
		return pgq_fail(PGQ_ERR_UNSUPPORTED, "iterativelengthbidirectional takes no flags and no sharding");
	}
	constexpr int W = 8; // LANE_LIMIT: a row's answer depends on the rows sharing its batch
	Run r(csr, ws, s);
	r.st.lanes = 64 * W;
	if (p == 0) {
		if (stats) {
			*stats = r.st;
		}
		return PGQ_OK;
	}
	CallCtx cc(p, d_src, d_dst, opts, d_out_len, d_out_valid);
	cc.ref_batching = true;
	// every row with a valid source and destination and src != dst takes a lane, in input order (l.93-116)
	LevelStatus *d_st = nullptr, *h_st = nullptr;
	PGQ_TRY(start_call<false>(r, cc, d_valid, 0, 0, 0, 1, &d_st, &h_st));
	const int total = h_st->total;
	int32_t *lane_dst;
	PGQ_TRY(pgq_ws_reserve(ws, WS_LANE_DST, (size_t)std::max(total, 1) * sizeof(int32_t), (void **)&lane_dst));
	k_lane_dst<<<grid_cap((p + 255) / 256, (int64_t)r.sms * 8), 256, 0, s>>>(p, cc.lm.row_lane, cc.lm.pdst, lane_dst);
	r.st.kernel_launches++;
	PGQ_CUDA(cudaGetLastError());
	const LaneMap lm_dst {cc.lm.row_lane, lane_dst, cc.lm.psrc, cc.lm.pdst, p};
	const int L = 64 * W;
	for (int pos = 0; pos < total; pos += L) {
		PGQ_TRY(run_bidir_batch<W>(r, cc, lm_dst, d_st, h_st, pos, std::min(L, total - pos)));
	}
	if (total == 0 || total % L == 0) {
		PGQ_TRY(count_empty_batch(r, cc.lm.row_lane, p));
	}
	return finish_call(r, stats);
}
