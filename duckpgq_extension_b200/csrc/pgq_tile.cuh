// pgq_tile.cuh -- device-side helpers shared by the CSR-build and BFS kernels.
#pragma once
#include "pgq_internal.h"

#define FULL_MASK 0xffffffffu

__device__ __forceinline__ uint32_t lanemask_le(int lane) {
	return 0xffffffffu >> (31 - lane);
}

// Walks one 256-position chunk of an adjacency array in 8 lane-strided steps and tells every
// lane which non-empty row (as a rank into DirGraph::nzrow) its position belongs to.
//   rank(e) = chunk_rank[c] - head_bit(256c) + popcount(head bits in [256c, e])
struct ChunkWalker {
	uint32_t hw;  // lane k (< 8) holds head word k of the chunk, lane 8 the first word of the next chunk
	int running;  // rank offset carried from the previous steps
	int64_t base; // first position of the chunk

	__device__ __forceinline__ ChunkWalker(const DirGraph &g, int64_t chunk, int lane) {
		hw = 1u;
		int r0 = 0;
		if (chunk < g.nchunks) {
			if (lane < PGQ_STEPS || (lane == PGQ_STEPS && chunk + 1 < g.nchunks)) {
				hw = g.head[chunk * PGQ_STEPS + lane];
			}
			r0 = g.chunk_rank[chunk];
		}
		base = chunk * PGQ_CHUNK;
		uint32_t h0 = __shfl_sync(FULL_MASK, hw, 0);
		running = r0 - (int)(h0 & 1u);
	}
	// head word of step k (bit i = position base + 32k + i starts a row)
	__device__ __forceinline__ uint32_t head_word(int k) const {
		return __shfl_sync(FULL_MASK, hw, k);
	}
	// rank of this lane's position in step k; call once per step, in order
	__device__ __forceinline__ int advance(uint32_t h, int lane) {
		int r = running + __popc(h & lanemask_le(lane));
		running += __popc(h);
		return r;
	}
};
