// pgq_count.cuh -- what the path-counting files share (pgq_allshortest.cu, pgq_kshortest.cu): saturating counts and
// the step-ordered in-lists.
#pragma once

#include "pgq_internal.h"

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
