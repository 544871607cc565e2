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
