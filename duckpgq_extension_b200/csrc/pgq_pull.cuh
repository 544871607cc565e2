// pgq_pull.cuh -- the fused bottom-up BFS level: expansion AND update in one pass over the in-edges.
//
//   next[n] = (OR_{(v -> n)} visit[v]) & ~seen[n];   seen[n] |= next[n]
//
// (iterativelength.cpp:18-30 of the reference with the loop nest turned inside out: rows = destinations.)
// Included by pgq_bfs.cu only (needs LaneMask / LevelStatus / ld_mask / st_mask / record_levels).
//
// The in-edges come in the layout the CSR build prepares for this kernel (PullGraph, pgq_internal.h):
//
//  LONG rows (in-degree >= 32) lie back to back in one adjacency array and are walked in RANGES of
//   4 chunks = 32 steps x 32 lanes = 1024 consecutive positions, one warp per range, ranges dealt
//   round-robin.  The OR of a row is kept LANE-DISTRIBUTED (every lane ORs the masks it gathered into
//   its own accumulator) for as long as the row lasts and is reduced across the warp (REDUX) once,
//   when the row ends: a hub row of 400 k in-edges costs one gather + four ORs per edge and a handful
//   of reductions.  A step holds at most ONE row head (rows are >= 32 long), so there is never a
//   segmented scan: lanes in front of the head finish the open row, lanes from the head on start the
//   next one.  Steps without a head take the fast path (G gathers in flight, no bookkeeping at all).
//
//  SHORT rows (in-degree 1..31: 86 % of the rows but 13 % of the edges of an R-MAT graph) are sorted
//   by degree and stored in SLICES of 32 rows, column-major (sliced ELL): lane l of the warp owns row l
//   of the slice, reads its j-th neighbour from column j (coalesced) and ORs the gathered masks in
//   registers -- no row heads, no shuffles, no reductions.
//
// In both parts the lane that holds a finished row's OR applies the level update on the spot (one
// 8W-byte load of seen, one store of the new frontier mask, one store of seen if anything is new):
// there is no separate dense update sweep and no second read of the candidate array.  The few long
// rows that cross a range boundary (at most one per range) are combined with atomicOr and finished
// by k_pull_finish.
//
// Finished rows: a search whose frontier has died out can never add a bit anywhere, so a destination
// that every LIVE lane has seen is finished for good; it is marked in a bitmap and from then on is
// neither gathered for nor written (k_pull_finish, pgq_bfs.cu, clears the two frontier entries it leaves
// behind), a range / slice whose rows are all finished costs one bitmap test, and a chunk inside a
// finished row is not even read.  (Undirected social graphs saturate after 3-4 levels; on directed
// R-MAT the levels behind the peak have 13 % and 0.1 % of the gathers left.)
//
// A row is always gathered to its end: stopping inside a row once the lanes that can still gain it are covered
// halved the gathers of the level behind the peak but saved no time, since the level is bound by the latency chains
// of its warps, not by the gathers alone.
#pragma once

#define PGQ_RANGE_CHUNKS 4
#define PGQ_RANGE_STEPS (PGQ_RANGE_CHUNKS * PGQ_STEPS)

template <int W>
struct PullArgs {
	PullGraph g;
	int64_t nranges;      // ranges of the long part
	int32_t gather_limit; // sources >= this cannot hold frontier bits in this level
	const u64 *visit;     // current frontier masks (read only)
	u64 *seen;
	u64 *cand;            // becomes the next frontier's visit array
	uint32_t *satbits;    // finished rows: bit k = long row of rank k, bit short_base + i = i-th short row
	int64_t short_base;
	int32_t *shared_row;  // [nranges] rank of the long row that ended in the range but began before it, or -1
	const int32_t *out_off;
	LevelStatus *st;
	uint16_t *level;
	int iter;
	int skip;
	// Finished rows are not written at all.  Their entries in the two mask buffers are zeroed behind the level by
	// k_pull_finish (bits newly set in the bitmap since the snapshot of two levels ago), so a range / slice whose rows
	// are all finished costs one or two loads of the bitmap and nothing else.
	LaneMask<W> live;
};

template <int W>
struct PullTotals {
	unsigned cnt = 0; // new frontier vertices
	unsigned gathers = 0; // mask gathers issued by this lane
	u64 edges = 0;    // their out-degrees
	u64 live[W];
	__device__ __forceinline__ PullTotals() {
#pragma unroll
		for (int i = 0; i < W; i++) {
			live[i] = 0;
		}
	}
};

// plain (coherent) mask load for arrays this kernel also writes: every row has one owner
template <int W>
__device__ __forceinline__ void ld_mask_rw(const u64 *base, int64_t idx, u64 (&m)[W]) {
	const u64 *p = base + idx * W;
	if constexpr (W == 1) {
		asm volatile("ld.global.u64 %0, [%1];" : "=l"(m[0]) : "l"(p));
	} else if constexpr (W == 2) {
		asm volatile("ld.global.v2.u64 {%0,%1}, [%2];" : "=l"(m[0]), "=l"(m[1]) : "l"(p));
	} else {
#pragma unroll
		for (int i = 0; i < W; i += 4) {
			PGQ_LD4("", p + i, m[i], m[i + 1], m[i + 2], m[i + 3]);
		}
	}
}

__device__ __forceinline__ bool sat_bit(const uint32_t *bits, int64_t k) {
	return (bits[k >> 5] >> (k & 31)) & 1u;
}

// The level update of one exclusive row (iterativelength.cpp:26-30): val = OR of the in-neighbours'
// frontier masks.  finished = the row was skipped because every live lane has seen it.  satpos = the
// row's bit in the finished-rows bitmap.
// (PATH: the discovery levels of the new bits are recorded here, by this one lane -- callers that have a whole
// warp at hand pass PATH = false and record cooperatively, record_levels_warp.)  On return val = the new bits.
template <int W, bool PATH>
__device__ __forceinline__ void pull_update_row(const PullArgs<W> &a, int row, u64 (&val)[W], bool finished,
                                                int64_t satpos, PullTotals<W> &tot) {
	if (finished) { // (both mask buffers hold zeros for it, or k_pull_finish is about to see to that)
#pragma unroll
		for (int i = 0; i < W; i++) {
			val[i] = 0;
		}
		return;
	}
	u64 sn[W];
	ld_mask_rw<W>(a.seen, row, sn);
	bool any_new = false, now_sat = true;
#pragma unroll
	for (int i = 0; i < W; i++) {
		val[i] &= ~sn[i];
		any_new |= val[i] != 0;
		sn[i] |= val[i];
		now_sat &= ((~sn[i]) & a.live.w[i]) == 0;
	}
	st_mask<W>(a.cand, row, val);
	if (any_new) {
		st_mask<W>(a.seen, row, sn);
		tot.cnt++;
		tot.edges += (u64)(a.out_off[row + 1] - a.out_off[row]);
#pragma unroll
		for (int i = 0; i < W; i++) {
			tot.live[i] |= val[i];
		}
		if (PATH) {
			record_levels<W>(val, row, a.level, a.iter);
		}
	}
	if (a.skip && now_sat) {
		atomicOr(&a.satbits[satpos >> 5], 1u << (satpos & 31));
	}
}

// path mode, long rows: lane 31 holds the row's new bits (val) after its update; the 32 lanes record the
// discovery level of two bits per mask word each (a hub row gains hundreds of bits in one level).
template <int W>
__device__ __forceinline__ void record_levels_warp(const PullArgs<W> &a, int row31, const u64 (&val31)[W], int lane) {
	const int row = __shfl_sync(FULL_MASK, row31, 31);
#pragma unroll
	for (int i = 0; i < W; i++) {
		const u64 word = __shfl_sync(FULL_MASK, val31[i], 31);
#pragma unroll
		for (int h = 0; h < 2; h++) {
			const int b = lane + 32 * h;
			if ((word >> b) & 1ull) {
				a.level[(int64_t)row * (64 * W) + 64 * i + b] = (uint16_t)a.iter; // (blind: see record_levels)
			}
		}
	}
}

template <int W>
__device__ __forceinline__ void pull_totals_flush(PullTotals<W> &tot, LevelStatus *st) {
	{
		const unsigned g = __reduce_add_sync(FULL_MASK, tot.gathers);
		if (g != 0 && (threadIdx.x & 31) == 0) {
			atomicAdd(&st->acc_gathers, (u64)g);
		}
	}
#pragma unroll
	for (int d = 16; d > 0; d >>= 1) {
		tot.cnt += __shfl_xor_sync(FULL_MASK, tot.cnt, d);
		tot.edges += __shfl_xor_sync(FULL_MASK, tot.edges, d);
	}
	if (tot.cnt == 0) { // (warp-uniform after the reduction)
		return;
	}
#pragma unroll
	for (int i = 0; i < W; i++) {
		tot.live[i] = warp_or(tot.live[i]);
	}
	if ((threadIdx.x & 31) == 0) {
		atomicAdd(&st->acc_vertices, (u64)tot.cnt);
		atomicAdd(&st->acc_edges, tot.edges);
#pragma unroll
		for (int i = 0; i < W; i++) {
			if (tot.live[i]) {
				atomicOr(&st->acc_live[i], tot.live[i]);
			}
		}
	}
}

// ---- one slice of 32 short rows: lane = row, column j = the rows' j-th in-neighbours ------------------------
template <int W, int G, bool PATH>
__device__ __forceinline__ void pull_short_slice(const PullArgs<W> &a, int64_t s, int lane, PullTotals<W> &tot) {
	const int64_t satpos = a.short_base + s * 32 + lane;
	bool fin = false;
	if (a.skip) { // the slice's 32 finished bits are one word of the bitmap (short_base is a multiple of 32)
		const uint32_t word = a.satbits[(a.short_base >> 5) + s];
		const int64_t left = a.g.n_short - s * 32;
		const uint32_t valid = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
		if ((word & valid) == valid) {
			return; // every row finished
		}
		fin = (word >> lane) & 1u;
	}
	const int row = a.g.s_row[s * 32 + lane]; // -1: the last slice is not full
	const int begin = a.g.s_off[s];
	const int width = (a.g.s_off[s + 1] - begin) >> 5;
	u64 acc[W];
#pragma unroll
	for (int i = 0; i < W; i++) {
		acc[i] = 0;
	}
	const int32_t *col = a.g.s_adj + begin + lane;
	for (int j0 = 0; j0 < width; j0 += G) {
		int u[G];
#pragma unroll
		for (int j = 0; j < G; j++) {
			u[j] = (j0 + j < width) ? col[(j0 + j) * 32] : -1;
		}
		u64 mv[G][W];
#pragma unroll
		for (int j = 0; j < G; j++) {
#pragma unroll
			for (int i = 0; i < W; i++) {
				mv[j][i] = 0;
			}
			if (!fin && (unsigned)u[j] < (unsigned)a.gather_limit) { // (padding is -1)
				tot.gathers++;
				ld_mask<W>(a.visit, u[j], mv[j]);
			}
		}
#pragma unroll
		for (int j = 0; j < G; j++) {
#pragma unroll
			for (int i = 0; i < W; i++) {
				acc[i] |= mv[j][i];
			}
		}
	}
	if (row >= 0) {
		pull_update_row<W, false>(a, row, acc, fin, satpos, tot); // acc becomes the row's new bits
	}
	if (PATH) { // the warp records the rows' discovery levels together, one row at a time (coalesced 2-byte stores)
		bool mine = false;
		if (row >= 0) {
#pragma unroll
			for (int i = 0; i < W; i++) {
				mine |= acc[i] != 0;
			}
		}
		unsigned todo = __ballot_sync(FULL_MASK, mine);
		while (todo) {
			const int src = __ffs(todo) - 1;
			todo &= todo - 1;
			const int r = __shfl_sync(FULL_MASK, row, src);
#pragma unroll
			for (int i = 0; i < W; i++) {
				const u64 word = __shfl_sync(FULL_MASK, acc[i], src);
#pragma unroll
				for (int h = 0; h < 2; h++) {
					const int b = lane + 32 * h;
					if ((word >> b) & 1ull) {
						a.level[(int64_t)r * (64 * W) + 64 * i + b] = (uint16_t)a.iter;
					}
				}
			}
		}
	}
}

// ---- one range of the long rows ---------------------------------------------------------------------------------
template <int W, int G, bool PATH>
__device__ __forceinline__ void pull_long_range(const PullArgs<W> &a, int64_t range, int lane, PullTotals<W> &tot) {
	const int64_t head_words = a.g.nchunks * PGQ_STEPS;
	const int64_t c0 = range * PGQ_RANGE_CHUNKS;
	const int64_t base = c0 * PGQ_CHUNK;
	if (a.skip) {
		// the rows that touch this range are the ranks kf .. kl (chunk_rank = rank of the row that covers a
		// chunk's first position): if all their finished bits are set there is nothing to do here
		const int64_t nc0 = c0 + PGQ_RANGE_CHUNKS;
		const int kf = a.g.chunk_rank[c0];
		const int kl = (nc0 >= a.g.nchunks) ? (int)a.g.n_rows - 1
		                                    : a.g.chunk_rank[nc0] - (int)(a.g.head[nc0 * PGQ_STEPS] & 1u);
		bool ok = true;
		for (int w0 = kf >> 5; w0 <= (kl >> 5); w0 += 32) {
			const int w = w0 + lane;
			if (w <= (kl >> 5)) {
				uint32_t need = 0xffffffffu;
				if (w == (kf >> 5)) {
					need &= 0xffffffffu << (kf & 31);
				}
				if (w == (kl >> 5)) {
					need &= 0xffffffffu >> (31 - (kl & 31));
				}
				ok &= (a.satbits[w] & need) == need;
			}
		}
		if (__all_sync(FULL_MASK, ok)) {
			if (lane == 31) {
				a.shared_row[range] = -1;
			}
			return;
		}
	}
	const int64_t hw_idx = c0 * PGQ_STEPS + lane;
	const uint32_t hw = (hw_idx < head_words) ? a.g.head[hw_idx] : 0u; // lane k: head word of step k
	const uint32_t headmask = __ballot_sync(FULL_MASK, hw != 0u);        // bit k: step k holds a row head
	// does the position right after the range start a row (or lie beyond the data)?
	const int64_t nc = c0 + PGQ_RANGE_CHUNKS;
	const bool next_head = (nc >= a.g.nchunks) ? true : ((a.g.head[nc * PGQ_STEPS] & 1u) != 0);
	const uint32_t h0 = __shfl_sync(FULL_MASK, hw, 0);
	int running = a.g.chunk_rank[c0] - (int)(h0 & 1u); // rank of the row that is open before the first position
	bool open_valid = !(h0 & 1u);                      // ... if the range does not start with a new row
	bool open_began = false;                           // did the open row begin inside this range?
	bool open_sat = false;                             // is it finished (no gathers needed)?
	if (a.skip && open_valid) {
		open_sat = sat_bit(a.satbits, running);
	}
	int shared = -1; // (lane 31) rank of the row that ends here but began in an earlier range
	u64 acc[W];
#pragma unroll
	for (int i = 0; i < W; i++) {
		acc[i] = 0;
	}
#pragma unroll 1
	for (int c = 0; c < PGQ_RANGE_CHUNKS; c++) {
		const int64_t cbase = base + (int64_t)c * PGQ_CHUNK;
		if (cbase >= a.g.m) {
			break;
		}
		const uint32_t chunk_heads = (headmask >> (c * PGQ_STEPS)) & 0xffu;
		if (chunk_heads == 0u && open_sat) {
			continue; // the whole chunk lies inside a finished row: its neighbour ids are not looked at
		}
		int u[PGQ_STEPS]; // the chunk's neighbour ids: 8 coalesced 128 B loads in flight
#pragma unroll
		for (int k = 0; k < PGQ_STEPS; k++) {
			const int64_t e = cbase + 32 * k + lane;
			u[k] = (e < a.g.m) ? a.g.adj[e] : -1;
		}
#pragma unroll
		for (int k0 = 0; k0 < PGQ_STEPS; k0 += G) {
			if (((chunk_heads >> k0) & ((1u << G) - 1u)) == 0u) {
				// ---- fast path: all G steps continue the open row
				if (!open_sat) {
					u64 mv[G][W];
#pragma unroll
					for (int j = 0; j < G; j++) {
#pragma unroll
						for (int i = 0; i < W; i++) {
							mv[j][i] = 0;
						}
						if ((unsigned)u[k0 + j] < (unsigned)a.gather_limit) {
							tot.gathers++;
							ld_mask<W>(a.visit, u[k0 + j], mv[j]);
						}
					}
#pragma unroll
					for (int j = 0; j < G; j++) {
#pragma unroll
						for (int i = 0; i < W; i++) {
							acc[i] |= mv[j][i];
						}
					}
				}
				continue;
			}
			// ---- a step of the group holds a row head (at most one per step: long rows have >= 32 edges)
			uint32_t hs[G];
			bool sat_new[G]; // is the row that starts in step j finished?
			{
				int r = running;
#pragma unroll
				for (int j = 0; j < G; j++) {
					hs[j] = __shfl_sync(FULL_MASK, hw, c * PGQ_STEPS + k0 + j);
					sat_new[j] = false;
					if (hs[j] != 0u) {
						r++;
						if (a.skip) {
							sat_new[j] = sat_bit(a.satbits, r);
						}
					}
				}
			}
			u64 mv[G][W];
			{
				bool cur_sat = open_sat;
#pragma unroll
				for (int j = 0; j < G; j++) {
					const uint32_t h = hs[j];
					const bool mine_sat = (h != 0u && lane >= __ffs(h) - 1) ? sat_new[j] : cur_sat;
#pragma unroll
					for (int i = 0; i < W; i++) {
						mv[j][i] = 0;
					}
					if (!mine_sat && (unsigned)u[k0 + j] < (unsigned)a.gather_limit) {
						tot.gathers++;
						ld_mask<W>(a.visit, u[k0 + j], mv[j]);
					}
					if (h != 0u) {
						cur_sat = sat_new[j];
					}
				}
			}
#pragma unroll
			for (int j = 0; j < G; j++) {
				const uint32_t h = hs[j];
				if (h == 0u) {
#pragma unroll
					for (int i = 0; i < W; i++) {
						acc[i] |= mv[j][i];
					}
					continue;
				}
				const int first = __ffs(h) - 1;
				if (lane < first) {
#pragma unroll
					for (int i = 0; i < W; i++) {
						acc[i] |= mv[j][i];
					}
				}
				if (open_valid && !open_sat) { // the open row ends in front of `first`: reduce it, lane 31 applies it
					u64 r[W];
#pragma unroll
					for (int i = 0; i < W; i++) {
						r[i] = warp_or(acc[i]);
					}
					int row31 = 0;
					if (lane == 31) {
						row31 = a.g.row[running];
						if (open_began) {
							pull_update_row<W, false>(a, row31, r, open_sat, running, tot); // r becomes the new bits
						} else { // began in an earlier range: combine, k_pull_finish applies the update
#pragma unroll
							for (int i = 0; i < W; i++) {
								if (r[i]) {
									atomicOr(&a.cand[(int64_t)row31 * W + i], r[i]);
								}
							}
							shared = running;
						}
					}
					if (PATH && open_began) { // (warp-uniform)
						record_levels_warp<W>(a, row31, r, lane);
					}
				}
				// the lanes from the head on start the new open row
				running++;
				open_valid = true;
				open_began = true;
				open_sat = sat_new[j];
#pragma unroll
				for (int i = 0; i < W; i++) {
					acc[i] = (lane >= first) ? mv[j][i] : 0;
				}
			}
		}
	}
	// ---- end of the range: the open row either ends here or continues in the next range
	if (open_valid && !open_sat) {
		u64 r[W];
#pragma unroll
		for (int i = 0; i < W; i++) {
			r[i] = warp_or(acc[i]);
		}
		int row31 = 0;
		if (lane == 31) {
			row31 = a.g.row[running];
			if (next_head && open_began) {
				pull_update_row<W, false>(a, row31, r, open_sat, running, tot); // r becomes the new bits
			} else {
#pragma unroll
				for (int i = 0; i < W; i++) {
					if (r[i]) {
						atomicOr(&a.cand[(int64_t)row31 * W + i], r[i]);
					}
				}
				if (next_head) {
					shared = running;
				}
			}
		}
		if (PATH && next_head && open_began) { // (warp-uniform)
			record_levels_warp<W>(a, row31, r, lane);
		}
	}
	if (lane == 31) {
		a.shared_row[range] = shared;
	}
}

// 256 threads per block, PGQ_PULL_CTAS blocks per SM: at most 80 registers per thread
#define PGQ_PULL_CTAS 3
template <int W, bool PATH>
__global__ void __launch_bounds__(256, PGQ_PULL_CTAS) k_pull_fused(const PullArgs<W> a) {
	// mask gathers in flight per lane: steps of a long-row range on the fast path, columns of a short-row slice
	constexpr int G = (W >= 8) ? 1 : ((W >= 4) ? 2 : 4);
	constexpr int GS = (W >= 8) ? 2 : 4;
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	PullTotals<W> tot;
	const int64_t items = a.nranges + a.g.n_slices;
	for (int64_t it = warp; it < items; it += nwarps) {
		if (it < a.nranges) {
			pull_long_range<W, G, PATH>(a, it, lane, tot);
		} else {
			pull_short_slice<W, GS, PATH>(a, it - a.nranges, lane, tot);
		}
	}
	pull_totals_flush<W>(tot, a.st);
}
