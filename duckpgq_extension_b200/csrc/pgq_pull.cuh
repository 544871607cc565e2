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
// EXIT (tuning variant 17, not the default): a row stops gathering inside a level once the lanes that
// can still gain it are covered.  Halves the gathers of the level behind the peak and saves no time.
#pragma once

#define PGQ_RANGE_CHUNKS 4
#define PGQ_RANGE_STEPS (PGQ_RANGE_CHUNKS * PGQ_STEPS)

template <int W>
struct PullArgs {
	PullGraph g;
	int64_t nranges;      // ranges of the long part
	int32_t gather_limit; // sources >= this cannot hold frontier bits in this level
	int32_t hub_limit;    // HINT variant: masks of sources below this are kept in L1 (evict_last), all others bypass it
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

// Mask gather with an L1 policy: the internal numbering puts the most gathered vertices first, so "u < hub_limit"
// are the few thousand masks that serve a quarter of all gathers -- they are asked to stay in L1 (evict_last) while
// every other mask, read about once per SM and level, does not allocate a line (no_allocate).
template <int W, int HINT>
__device__ __forceinline__ void ld_mask_hint(const u64 *__restrict__ base, int64_t idx, u64 (&m)[W], bool hot) {
	const u64 *p = base + idx * W;
	if constexpr (W == 4 && HINT == 1) {
		if (hot) {
			PGQ_LD4(".nc.L1::evict_last", p, m[0], m[1], m[2], m[3]);
		} else {
			PGQ_LD4(".nc.L1::no_allocate", p, m[0], m[1], m[2], m[3]);
		}
	} else if constexpr (W >= 4 && HINT == 2) { // (experiment: L2 eviction priorities on top, 32 B masks and wider only)
		// sm_90 takes an L2 eviction priority only as a cache policy (createpolicy) handed to the load
		u64 pol;
		if (hot) {
			asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
		} else {
			asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
		}
#pragma unroll
		for (int i = 0; i < W; i += 4) {
			if (hot) {
				asm volatile("ld.global.nc.L1::evict_last.L2::cache_hint.v2.u64 {%0,%1}, [%4], %5;\n\t"
				             "ld.global.nc.L1::evict_last.L2::cache_hint.v2.u64 {%2,%3}, [%4+16], %5;"
				             : "=&l"(m[i]), "=&l"(m[i + 1]), "=&l"(m[i + 2]), "=&l"(m[i + 3])
				             : "l"(p + i), "l"(pol));
			} else {
				asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0,%1}, [%4], %5;\n\t"
				             "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%2,%3}, [%4+16], %5;"
				             : "=&l"(m[i]), "=&l"(m[i + 1]), "=&l"(m[i + 2]), "=&l"(m[i + 3])
				             : "l"(p + i), "l"(pol));
			}
		}
	} else if constexpr (HINT == 3) { // hub masks staged in shared memory (k_pull_fused_hub), all others bypass L1
		if (hot) {
			extern __shared__ __align__(128) unsigned char pull_smem[];
			const u64 *q = reinterpret_cast<const u64 *>(pull_smem) + idx * W;
			if constexpr (W == 1) {
				m[0] = q[0];
			} else {
#pragma unroll
				for (int i = 0; i < W; i += 2) {
					const ulonglong2 t = *reinterpret_cast<const ulonglong2 *>(q + i);
					m[i] = t.x;
					m[i + 1] = t.y;
				}
			}
		} else if constexpr (W == 1) {
			asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(m[0]) : "l"(p));
		} else if constexpr (W == 2) {
			asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%2];" : "=l"(m[0]), "=l"(m[1]) : "l"(p));
		} else {
#pragma unroll
			for (int i = 0; i < W; i += 4) {
				PGQ_LD4(".nc.L1::no_allocate", p + i, m[i], m[i + 1], m[i + 2], m[i + 3]);
			}
		}
	} else {
		ld_mask<W>(base, idx, m);
	}
}

__device__ __forceinline__ int ld_adj_stream(const int32_t *p) { // the 4 B/edge stream: read once, never again
	int v;
	asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
	return v;
}

__device__ __forceinline__ bool sat_bit(const uint32_t *bits, int64_t k) {
	return (bits[k >> 5] >> (k & 31)) & 1u;
}

// The level update of one exclusive row (iterativelength.cpp:26-30): val = OR of the in-neighbours'
// frontier masks.  finished = the row was skipped because every live lane has seen it.  satpos = the
// row's bit in the finished-rows bitmap.
// (PATH: the discovery levels of the new bits are recorded here, by this one lane -- callers that have a whole
// warp at hand pass PATH = false and record cooperatively, record_levels_warp.)  On return val = the new bits.
template <int W, bool PATH, bool HAVE_SEEN = false>
__device__ __forceinline__ void pull_update_row(const PullArgs<W> &a, int row, u64 (&val)[W], bool finished,
                                                int64_t satpos, PullTotals<W> &tot, u64 *seen_row = nullptr) {
	if (finished) { // (both mask buffers hold zeros for it, or k_pull_finish is about to see to that)
#pragma unroll
		for (int i = 0; i < W; i++) {
			val[i] = 0;
		}
		return;
	}
	u64 sn[W];
	if constexpr (HAVE_SEEN) {
#pragma unroll
		for (int i = 0; i < W; i++) {
			sn[i] = seen_row[i];
		}
	} else {
		ld_mask_rw<W>(a.seen, row, sn);
	}
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
template <int W, int G, bool PATH, int HINT, bool EXIT = false>
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
	// EXIT: the lane's row can gain only the bits need = live & ~seen (a lane whose frontier is empty has no bit
	// in any visit mask); once the gathered OR covers them, the rest of the row cannot change the result.
	u64 sn[W];
	bool full = false; // early exit reached: no more gathers for this lane's row
	if constexpr (EXIT) {
		if (!fin && row >= 0) {
			ld_mask_rw<W>(a.seen, row, sn);
		} else {
#pragma unroll
			for (int i = 0; i < W; i++) {
				sn[i] = ~0ull;
			}
		}
	}
	{
		const int32_t *col = a.g.s_adj + begin + lane;
		for (int j0 = 0; j0 < width; j0 += G) {
			if constexpr (EXIT) {
				if (__all_sync(FULL_MASK, fin || full || row < 0)) {
					break;
				}
			}
			int u[G];
#pragma unroll
			for (int j = 0; j < G; j++) {
				u[j] = (j0 + j < width) ? (HINT != 0 ? ld_adj_stream(col + (j0 + j) * 32) : col[(j0 + j) * 32]) : -1;
			}
			u64 mv[G][W];
#pragma unroll
			for (int j = 0; j < G; j++) {
#pragma unroll
				for (int i = 0; i < W; i++) {
					mv[j][i] = 0;
				}
				if (!fin && !(EXIT && full) && (unsigned)u[j] < (unsigned)a.gather_limit) { // (padding is -1)
					tot.gathers++;
					if constexpr (HINT != 0) {
						ld_mask_hint<W, HINT>(a.visit, u[j], mv[j], u[j] < a.hub_limit);
					} else {
						ld_mask<W>(a.visit, u[j], mv[j]);
					}
				}
			}
#pragma unroll
			for (int j = 0; j < G; j++) {
#pragma unroll
				for (int i = 0; i < W; i++) {
					acc[i] |= mv[j][i];
				}
			}
			if constexpr (EXIT) {
				bool covered = true;
#pragma unroll
				for (int i = 0; i < W; i++) {
					covered &= (a.live.w[i] & ~sn[i] & ~acc[i]) == 0;
				}
				full = covered;
			}
		}
	}
	if (row >= 0) {
		if constexpr (EXIT) {
			pull_update_row<W, false, true>(a, row, acc, fin, satpos, tot, sn); // acc becomes the row's new bits
		} else {
			pull_update_row<W, false>(a, row, acc, fin, satpos, tot);
		}
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

// ---- bulk async copies (TMA engine, cp.async.bulk -> UBLKCP) of the neighbour-id stream into shared memory ------
// A warp keeps two 1 KB stages: while it gathers for one chunk (256 neighbour ids), the copy engine brings its
// next chunk in, so the only global loads the warp itself issues for the long rows are the mask gathers.
#define PGQ_CHUNK_BYTES (PGQ_CHUNK * 4)

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
	return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
}
// one lane: announce the bytes, start the copy global -> shared; completion arrives on the barrier
__device__ __forceinline__ void bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
	             "l"(src), "r"(bytes), "r"(smem_u32(bar))
	             : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
	asm volatile("{\n"
	             ".reg .pred p;\n"
	             "WAIT_%=:\n"
	             "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
	             "@p bra DONE_%=;\n"
	             "bra WAIT_%=;\n"
	             "DONE_%=:\n"
	             "}" ::"r"(smem_u32(bar)),
	             "r"(parity)
	             : "memory");
}

struct AdjPipe {
	int32_t *stage = nullptr; // two stages of PGQ_CHUNK ids; nullptr = no staging (plain LDG)
	uint64_t *bar = nullptr;
	uint32_t parity0 = 0, parity1 = 0;
	int cur = 0;
};

// ---- one range of the long rows ---------------------------------------------------------------------------------
template <int W, int G, bool PATH, bool BULK, int HINT, bool EXIT = false>
__device__ __forceinline__ void pull_long_range(const PullArgs<W> &a, int64_t range, int64_t next_range, int lane,
                                                PullTotals<W> &tot, AdjPipe &pipe) {
	const int64_t head_words = a.g.nchunks * PGQ_STEPS;
	const int64_t c0 = range * PGQ_RANGE_CHUNKS;
	const int64_t base = c0 * PGQ_CHUNK;
	if constexpr (!BULK) {
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
	// EXIT: lane i < W holds word i of need = live & ~seen[open row] from the row's first head-less group on;
	// once the warp's gathered OR covers it, the rest of the row (inside this range) is not gathered any more.
	bool open_full = false, need_valid = false;
	u64 need_word = 0;
	if constexpr (EXIT) {
		// A range that starts deep inside a row (no head in its first chunk) is a continuation range of a hub row:
		// the kernel runs those after all others, so the ranges in front of it have usually published their part
		// of the row's OR in cand already -- what they found need not be found again, and if nothing is missing the
		// whole open part is skipped.  (Stale or partial values of cand only make the test more conservative.)
		if (open_valid && !open_sat && (headmask & 0xffu) == 0u) {
			const int orow = a.g.row[running];
			const int wsel = lane & (W - 1);
			u64 lw = a.live.w[0];
#pragma unroll
			for (int i = 1; i < W; i++) {
				lw = (wsel == i) ? a.live.w[i] : lw;
			}
			const u64 sw = __ldcg(a.seen + (int64_t)orow * W + wsel);
			const u64 cw = __ldcg(a.cand + (int64_t)orow * W + wsel);
			need_word = lw & ~sw & ~cw;
			need_valid = true;
			open_full = !__any_sync(FULL_MASK, need_word != 0);
		}
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
		const int32_t *staged = nullptr;
		if constexpr (BULK) {
			// the copy of THIS chunk was started one chunk ago; start the copy of the warp's next chunk, then wait
			int64_t nbase = cbase + PGQ_CHUNK; // next chunk of this range ...
			if (c + 1 == PGQ_RANGE_CHUNKS || nbase >= a.g.m) {
				nbase = (next_range >= 0) ? next_range * PGQ_RANGE_CHUNKS * PGQ_CHUNK : -1; // ... or the first of the next one
			}
			__syncwarp(); // every lane is done reading the stage that is about to be overwritten
			if (nbase >= 0 && lane == 0) {
				asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
				bulk_load(pipe.stage + (pipe.cur ^ 1) * PGQ_CHUNK, a.g.adj + nbase, PGQ_CHUNK_BYTES, &pipe.bar[pipe.cur ^ 1]);
			}
			if (pipe.cur == 0) {
				mbar_wait(&pipe.bar[0], pipe.parity0);
				pipe.parity0 ^= 1u;
			} else {
				mbar_wait(&pipe.bar[1], pipe.parity1);
				pipe.parity1 ^= 1u;
			}
			staged = pipe.stage + pipe.cur * PGQ_CHUNK;
			pipe.cur ^= 1;
		}
		if (chunk_heads == 0u && (open_sat || (EXIT && open_full))) {
			continue; // the whole chunk lies inside a finished row: its neighbour ids are not looked at
		}
		int u[PGQ_STEPS]; // the chunk's neighbour ids: 8 coalesced 128 B loads in flight, or 8 LDS from the stage
#pragma unroll
		for (int k = 0; k < PGQ_STEPS; k++) {
			const int64_t e = cbase + 32 * k + lane;
			if constexpr (BULK) {
				u[k] = (e < a.g.m) ? staged[32 * k + lane] : -1;
			} else {
				u[k] = (e < a.g.m) ? (HINT != 0 ? ld_adj_stream(a.g.adj + e) : a.g.adj[e]) : -1;
			}
		}
#pragma unroll
		for (int k0 = 0; k0 < PGQ_STEPS; k0 += G) {
			if (((chunk_heads >> k0) & ((1u << G) - 1u)) == 0u) {
				// ---- fast path: all G steps continue the open row
				if (!open_sat && !(EXIT && open_full)) {
					if constexpr (EXIT) {
						if (!need_valid) { // (in flight together with the gathers below)
							const int orow = a.g.row[running];
							const int wsel = lane & (W - 1);
							u64 sw, lw = a.live.w[0];
							asm volatile("ld.global.u64 %0, [%1];" : "=l"(sw) : "l"(a.seen + (int64_t)orow * W + wsel));
#pragma unroll
							for (int i = 1; i < W; i++) {
								lw = (wsel == i) ? a.live.w[i] : lw;
							}
							need_word = lw & ~sw;
							need_valid = true;
						}
					}
					u64 mv[G][W];
#pragma unroll
					for (int j = 0; j < G; j++) {
#pragma unroll
						for (int i = 0; i < W; i++) {
							mv[j][i] = 0;
						}
						if ((unsigned)u[k0 + j] < (unsigned)a.gather_limit) {
							tot.gathers++;
							if constexpr (HINT != 0) {
								ld_mask_hint<W, HINT>(a.visit, u[k0 + j], mv[j], u[k0 + j] < a.hub_limit);
							} else {
								ld_mask<W>(a.visit, u[k0 + j], mv[j]);
							}
						}
					}
#pragma unroll
					for (int j = 0; j < G; j++) {
#pragma unroll
						for (int i = 0; i < W; i++) {
							acc[i] |= mv[j][i];
						}
					}
					if constexpr (EXIT) {
						u64 mine = 0; // word (lane & (W-1)) of the warp's OR so far
#pragma unroll
						for (int i = 0; i < W; i++) {
							const u64 f = warp_or(acc[i]);
							mine = ((lane & (W - 1)) == i) ? f : mine;
						}
						open_full = !__any_sync(FULL_MASK, (need_word & ~mine) != 0);
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
				bool cur_sat = open_sat || (EXIT && open_full);
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
						if constexpr (HINT != 0) {
							ld_mask_hint<W, HINT>(a.visit, u[k0 + j], mv[j], u[k0 + j] < a.hub_limit);
						} else {
							ld_mask<W>(a.visit, u[k0 + j], mv[j]);
						}
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
				open_full = false;
				need_valid = false;
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

template <int W, int G, int MB, bool PATH, bool BULK, int HINT = 0, bool EXIT = false>
__global__ void __launch_bounds__(256, MB) k_pull_fused(const PullArgs<W> a) {
	extern __shared__ __align__(128) unsigned char pull_smem[]; // BULK: per warp two 1 KB stages, then the barriers
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	PullTotals<W> tot;
	AdjPipe pipe;
	if constexpr (BULK) {
		const int wib = threadIdx.x >> 5;
		pipe.stage = reinterpret_cast<int32_t *>(pull_smem) + wib * 2 * PGQ_CHUNK;
		pipe.bar = reinterpret_cast<uint64_t *>(pull_smem + 8 * 2 * PGQ_CHUNK_BYTES) + wib * 2;
		if (lane == 0) {
			mbar_init(&pipe.bar[0]);
			mbar_init(&pipe.bar[1]);
			asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
			if (warp < a.nranges) { // the first chunk of the warp's first range
				bulk_load(pipe.stage, a.g.adj + warp * PGQ_RANGE_CHUNKS * PGQ_CHUNK, PGQ_CHUNK_BYTES, &pipe.bar[0]);
			}
		}
		__syncwarp();
	}
	const int64_t items = a.nranges + a.g.n_slices;
	if constexpr (EXIT && !BULK) {
		// pass 0: the ranges with a row head in their first chunk; pass 1: continuation ranges of hub rows (see
		// pull_long_range); then the short rows
		// (work is handed out by tickets: rows that exit early make the ranges very unequal)
		const int64_t head_words = a.g.nchunks * PGQ_STEPS;
		for (int pass = 0; pass < 2; pass++) {
			for (;;) {
				unsigned t = 0;
				if (lane == 0) {
					t = atomicAdd(&a.st->pull_ticket[pass], 1u);
				}
				const int64_t it = __shfl_sync(FULL_MASK, t, 0);
				if (it >= a.nranges) {
					break;
				}
				const int64_t hi = it * PGQ_RANGE_STEPS + lane;
				const uint32_t w0 = (lane < PGQ_STEPS && hi < head_words) ? a.g.head[hi] : 0u;
				const int cls = __any_sync(FULL_MASK, w0 != 0u) ? 0 : 1;
				if (cls == pass) {
					pull_long_range<W, G, PATH, BULK, HINT, EXIT>(a, it, -1, lane, tot, pipe);
				}
			}
		}
		for (;;) {
			unsigned t = 0;
			if (lane == 0) {
				t = atomicAdd(&a.st->pull_ticket[2], 1u);
			}
			const int64_t it = __shfl_sync(FULL_MASK, t, 0);
			if (it >= a.g.n_slices) {
				break;
			}
			pull_short_slice<W, (W >= 8 ? 2 : 4), PATH, HINT, EXIT>(a, it, lane, tot);
		}
	} else {
		for (int64_t it = warp; it < items; it += nwarps) {
			if (it < a.nranges) {
				const int64_t nxt = (it + nwarps < a.nranges) ? it + nwarps : -1;
				pull_long_range<W, G, PATH, BULK, HINT, EXIT>(a, it, nxt, lane, tot, pipe);
			} else {
				pull_short_slice<W, (W >= 8 ? 2 : 4), PATH, HINT, EXIT>(a, it - a.nranges, lane, tot);
			}
		}
	}
	pull_totals_flush<W>(tot, a.st);
}

// The same level with the masks of the first `hub_limit` vertices of the internal numbering -- the most gathered
// ones: on R-MAT-22 the first 7168 serve 32 % of all gathers -- staged in shared memory: one CTA of 24 warps per SM
// copies them in (coalesced, 224 KB) and serves those gathers with LDS instead of an L1-missing sector request.
#define PGQ_HUB_SMEM_BYTES 229376
template <int W, int G, bool PATH>
__global__ void __launch_bounds__(768, 1) k_pull_fused_hub(const PullArgs<W> a) {
	extern __shared__ __align__(128) unsigned char pull_smem[];
	{
		const uint4 *from = reinterpret_cast<const uint4 *>(a.visit);
		uint4 *to = reinterpret_cast<uint4 *>(pull_smem);
		const int n16 = a.hub_limit * W / 2;
		for (int i = threadIdx.x; i < n16; i += blockDim.x) {
			to[i] = __ldg(from + i);
		}
	}
	__syncthreads();
	const int lane = threadIdx.x & 31;
	const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
	PullTotals<W> tot;
	AdjPipe pipe;
	const int64_t items = a.nranges + a.g.n_slices;
	for (int64_t it = warp; it < items; it += nwarps) {
		if (it < a.nranges) {
			pull_long_range<W, G, PATH, false, 3>(a, it, -1, lane, tot, pipe);
		} else {
			pull_short_slice<W, (W >= 8 ? 2 : 4), PATH, 3>(a, it - a.nranges, lane, tot);
		}
	}
	pull_totals_flush<W>(tot, a.st);
}
