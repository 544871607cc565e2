// pgq_kpaths.cuh -- the rounds of Yen's algorithm with Lawler's rule (km_run, pgq_kpaths_modes.cu's top), shared by the
// calls that run them over a spur search of their own: shortest_k_paths_mode and shortest_k_groups with a BFS
// (pgq_kpaths_modes.cu), cheapest_k_paths with a Bellman-Ford (pgq_cheapest_k.cu).
#pragma once

#include <algorithm>
#include <vector>

#include "pgq_internal.h"
#include "pgq_tile.cuh"

#define KM_PATH_MAX 65533 // the longest path a result may hold (all_shortest_paths' depth limit)

// One spur search: its spur node and target (internal ids) and its ban lists in the round's list array: vb the banned
// vertices (internal ids), d the deviation bans and eb the banned edges (out-CSR positions)
struct KmSpur {
	int32_t u, t, nvb, nd, neb, pad;
	int64_t vb, d, eb;
};

__device__ __forceinline__ bool km_in(const int32_t *__restrict__ list, int cnt, int32_t x) {
	for (int i = 0; i < cnt; i++) {
		if (list[i] == x) {
			return true;
		}
	}
	return false;
}

// entry e (to v) of u's adjacency may start the spur
__device__ __forceinline__ bool km_first_ok(const KmSpur &sp, const int32_t *__restrict__ lists, int32_t e, int32_t v) {
	return !km_in(lists + sp.d, sp.nd, e) && !km_in(lists + sp.eb, sp.neb, e) && !km_in(lists + sp.vb, sp.nvb, v);
}

// the lanes whose banned positions include e, within mask word j: keys sorted, key = position * 512 + lane
__device__ __forceinline__ u64 km_ban_mask(const int64_t *__restrict__ keys, int64_t nkeys, int64_t e, int j) {
	int64_t lo = 0, hi = nkeys;
	while (lo < hi) {
		const int64_t mid = (lo + hi) >> 1;
		if (keys[mid] < e * 512) {
			lo = mid + 1;
		} else {
			hi = mid;
		}
	}
	u64 mask = 0;
	for (; lo < nkeys && (keys[lo] >> 9) == e; lo++) {
		const int l = (int)(keys[lo] & 511);
		if ((l >> 6) == j) {
			mask |= 1ull << (l & 63);
		}
	}
	return mask;
}

// One batch of a round as km_run hands it to the spur search: cnt lanes in a batch W wide, lane l searching spur
// lane_spur[l] of the round's spurs; TRAIL's banned positions as a bitmap over out-CSR positions and the sorted
// (position * 512 + lane) table (both null when the batch bans none).  The search leaves each lane's spur length in
// hlen (device) and h_hlen (host), 0 for no spur.
struct KmBatch {
	int cnt, W;
	unsigned lane_grid; // a warp per lane
	const int32_t *lane_spur;
	const KmSpur *spurs;
	const int32_t *lists;
	uint32_t *ban_bits;
	const int64_t *keys;
	int64_t nkeys;
	int32_t *hlen, *h_hlen;
};

// The spur search of km_run's rounds.  cap is the call's widest lane width, lane_min the narrowest a round halves it
// to; with `costs` the paths carry their costs (the sums of their weights), which lead the pool's key.
struct KmSearch {
	int cap = 0, lane_min = 64;
	bool costs = false;
	// reserves the call's buffers for cap lanes, behind the step lists
	virtual int begin(Workspace *ws, const u64 *step_key, const int32_t *step_pos) = 0;
	// has[x] = spur x of the round has an admissible first edge (device); root[x] = the cost of its root (with costs)
	virtual int has_seed(Workspace *ws, int64_t ns, const KmSpur *spurs, const int32_t *lists,
	                     const std::vector<int64_t> &root, uint8_t *has, pgq_stats *st) = 0;
	// searches a batch's lanes: hlen and h_hlen
	virtual int search(Workspace *ws, const KmBatch &b, pgq_stats *st) = 0;
	// walks the found spurs of the batch back: step i of lane l (0 = the edge out of u) goes to steps[lane_off[l] + i]
	// as (parent's internal id, out-CSR position) and to step_elems as (parent's original id, edge rowid); with costs,
	// the edge's weight bits to step_w
	virtual int walk(Workspace *ws, const KmBatch &b, const int64_t *lane_off, int2 *steps, longlong2 *step_elems,
	                 int64_t *step_w, pgq_stats *st) = 0;
};

struct KmGroups;

// The rounds (pgq_kpaths_modes.cu's top) over `search`, for shortest_k_paths_mode (kg null), shortest_k_groups and
// cheapest_k_paths (out_costs non-null: each path's cost as raw weight bits, allocated like the other arrays).  The
// arguments are checked.
int km_run(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
           const uint8_t *dst_valid, const pgq_options *opts, int64_t k, int32_t path_mode, const KmGroups *kg,
           KmSearch &search, int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
           int64_t **out_path_offsets, int64_t **out_elems, void **out_costs, int64_t *out_total_paths,
           pgq_stats *stats);
