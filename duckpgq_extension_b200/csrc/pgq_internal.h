// pgq_internal.h -- shared host-side declarations of libduckpgq_b200 (not part of the C ABI).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <condition_variable>
#include <map>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <string>
#include <vector>

#include "duckpgq_b200.h"

typedef unsigned long long u64;

// ---- error plumbing: nothing throws across the C ABI -------------------------------------------
void pgq_set_error(const char *fmt, ...);
int pgq_fail(int status, const char *fmt, ...);

#define PGQ_CUDA(call)                                                                                      \
	do {                                                                                                    \
		cudaError_t _e = (call);                                                                            \
		if (_e != cudaSuccess) {                                                                            \
			cudaGetLastError();                                                                             \
			return pgq_fail(_e == cudaErrorMemoryAllocation ? PGQ_ERR_OOM : PGQ_ERR_CUDA, "%s failed: %s (%s:%d)", \
			                #call, cudaGetErrorString(_e), __FILE__, __LINE__);                             \
		}                                                                                                   \
	} while (0)

#define PGQ_TRY(call)           \
	do {                        \
		int _s = (call);        \
		if (_s != PGQ_OK) {     \
			return _s;          \
		}                       \
	} while (0)

// a launch's grid: want blocks, at least 1 and at most cap
static inline unsigned grid_size(int64_t want, int64_t cap) {
	return (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, cap));
}

// ---- geometry of the edge-tiled kernels --------------------------------------------------------
// A "chunk" is 256 consecutive positions of an adjacency array, processed by one warp as 8 steps
// of 32 lane-strided edges (perfectly coalesced 128 B loads).  Which row (vertex) an edge belongs
// to is recovered from a 1-bit-per-edge row-head bitmap plus one rank per chunk, so the kernels
// never binary-search the offsets and never see empty rows.
#define PGQ_CHUNK 256
#define PGQ_STEPS 8

// One direction of the graph: the out-CSR (row = source) or the in-CSC (row = destination).  Only the out-CSR has
// head / nzrow / chunk_rank (the edge-tiled CSR build kernels walk it); the in-CSC is off / adj alone, and nnz /
// nchunks are 0 there.
struct DirGraph {
	int32_t *off = nullptr;        // [n+1] row offsets
	int32_t *adj = nullptr;        // [m]   neighbour ids
	uint32_t *head = nullptr;      // [nchunks*8] bit e = 1 iff position e is the first of its row
	int32_t *nzrow = nullptr;      // [nnz] ids of the non-empty rows, ascending
	int32_t *chunk_rank = nullptr; // [nchunks] index into nzrow of the row holding position 256*c
	int64_t nnz = 0;
	int64_t nchunks = 0;
};

// The in-edges in the layout of the fused bottom-up level (pgq_pull.cuh), built once per CSR next to the
// plain in-CSC (which path reconstruction keeps using):
//   long rows  (in-degree >= PGQ_SHORT_DEG): in-lists back to back in row order + head bitmap + chunk ranks;
//              `row` maps the rank of a long row to its vertex id
//   short rows (in-degree 1 .. PGQ_SHORT_DEG - 1): sorted by descending degree (ties by id), in slices of 32
//              rows stored column-major: s_adj[s_off[s] + j * 32 + l] = j-th in-neighbour of the slice's l-th row
//              (-1 = padding), s_row[s * 32 + l] = that row's vertex id (-1 = none)
#define PGQ_SHORT_DEG 32
struct PullGraph {
	int32_t *adj = nullptr;
	uint32_t *head = nullptr;
	int32_t *chunk_rank = nullptr;
	int32_t *row = nullptr;
	int64_t m = 0, nchunks = 0, n_rows = 0;
	int32_t *s_adj = nullptr;
	int32_t *s_row = nullptr;
	int32_t *s_off = nullptr;
	int64_t n_short = 0, n_slices = 0, s_total = 0;
};

// ---- workspace slots ---------------------------------------------------------------------------
// A workspace holds one device buffer per slot.  The blocks below say who holds a slot and for how long.  Consumers
// that never run at the same time on one workspace share numbers on purpose, so that a pooled workspace holds the
// largest of their buffers rather than the sum: one number may have a name in several blocks.
enum WsSlot : int {
	// The search masks, persistent across calls: a workspace remembers which of their rows hold zeros
	// (Workspace::clean_from), so only the BFS drivers may write them.
	WS_SEEN = 28, WS_VISIT_A = 29, WS_VISIT_B = 30,
	// radix_sort_pairs' histogram and scan scratch: a caller of it keeps nothing here.
	WS_RADIX_HIST = 14, WS_RADIX_SCAN = 15,
	// The host columns of the path entry points (pgq_api.cu, pgq_cheapest.cu) staged on the device, and their results
	// there.  They live while a driver runs, so no driver uses them.  (WS_OUT_OFFSETS is shortestpath's,
	// WS_IN_DST_VALID cheapest_path_length's and cheapest_path's; cheapest_path keeps its costs in WS_OUT_LEN / _VALID
	// and returns its lists in WS_OUT_PATH_OFFSETS, WS_OUT_LENGTHS and WS_OUT_PATH_VALID.)
	WS_IN_SRC = 6, WS_IN_DST = 7, WS_IN_VALID = 8, WS_OUT_LEN = 9, WS_OUT_VALID = 10, WS_OUT_OFFSETS = 11,
	WS_IN_DST_VALID = 11, WS_OUT_LENGTHS = 12, WS_OUT_PATH_OFFSETS = 31, WS_OUT_PATH_VALID = 39,
	// The BFS call driver (pgq_bfs.cu), then the second side of iterativelengthbidirectional: its masks, item lists,
	// lane -> seed vertex map and the meet test's accumulator.  (A bidirectional call leaves the search masks dirty
	// outside the known-zero rows, and says so through Workspace::clean_from.)
	WS_ROW_LANE = 3, WS_STATUS = 4, WS_LEVEL = 5, WS_ITEMS_A = 13, WS_ITEMS_B = 14, WS_TLIST = 15, WS_TBITS = 16,
	WS_WALK = 17, WS_ELEMS = 18, WS_SLOT_OFF = 19, WS_PSRC = 20, WS_PDST = 21, WS_SATBITS = 22, WS_SHARED_ROWS = 23,
	WS_LANE_SRC = 24, WS_ASSIGN_TMP = 25, WS_BATCH_ROWS = 26, WS_PATH_TOTAL = 27,
	WS_SEEN_D = 32, WS_VISIT_A_D = 33, WS_VISIT_B_D = 34, WS_LANE_DST = 35, WS_ITEMS_A_D = 36, WS_ITEMS_B_D = 37,
	WS_MEET = 38,
	// Scratch of the CSR build (finalize, metadata, bottom-up layout, upload) and of the downloads: a scan's scratch,
	// the error flag, small flags, an int64 column, O(n + m) temporaries (the sorts' buffers, a download's second
	// column) and per-vertex arrays.
	WS_CSR_SCAN = 1, WS_CSR_ERR = 2, WS_CSR_FLAGS = 3, WS_CSR_WIDE = 4, WS_CSR_EDGE_A = 5, WS_CSR_EDGE_B = 6,
	WS_CSR_EDGE_C = 7, WS_CSR_VERTEX_A = 0, WS_CSR_VERTEX_B = 9, WS_CSR_VERTEX_C = 10, WS_CSR_VERTEX_D = 11,
	WS_CSR_VERTEX_E = 12,
	// cheapest_path_length (pgq_cheapest.cu)
	WS_BF_DIST = 0, WS_BF_DIRTY = 1, WS_BF_FLAGS = 2,
	// cheapest_path's tight search, behind each batch's sweeps (pgq_cheapest.cu): the levels h, the parent keys, the
	// two frontier maps, each lane's target and the level counters; the lists go to shortestpath's element array
	// (WS_ELEMS), the element count of a batch's rows to WS_PATH_TOTAL.
	WS_CP_LEVEL = 3, WS_CP_PKEY = 4, WS_CP_FRONTIER = 5, WS_CP_LANE_TGT = 13, WS_CP_COUNTERS = 15,
	// local_clustering_coefficient: its staged column and results
	WS_LCC_SRC = 16, WS_LCC_OUT = 17, WS_LCC_OUT_VALID = 18, WS_LCC_BIG_ROWS = 19, WS_LCC_BIG_CNT = 20,
	WS_LCC_SRC_VALID = 21, WS_LCC_BITMAP = 22,
	// pagerank and weakly_connected_component.  WCC's six edge arrays take WS_WCC_EDGES and the five slots after it;
	// its merge sort reuses the first three once they are dead.
	WS_AN_REF_OFF = 16, WS_AN_SCAN = 17, WS_PR_KEY_A = 18, WS_PR_KEY_B = 19, WS_PR_VAL_A = 20, WS_PR_VAL_B = 21,
	WS_PR_IN_OFF = 22, WS_PR_SCAN = 23, WS_PR_DFLAG = 24, WS_PR_RANK = 25, WS_PR_TEMP = 26, WS_PR_CONTRIB = 27,
	WS_PR_DANGLING = 12, WS_PR_TOTAL = 13,
	WS_WCC_EDGES = 18, WS_WCC_COMP = 24, WS_WCC_HOOK = 25, WS_WCC_BEST = 26, WS_WCC_MERGE_POS = 27, WS_WCC_MERGE_A = 11,
	WS_WCC_MERGE_B = 12, WS_WCC_FLAGS = 13, WS_WCC_SORT_KEY = 18, WS_WCC_SORT_IDX_A = 19, WS_WCC_SORT_IDX_B = 20,
	// The key builds (pgq_csr_build_keys*), which go on into the CSR build's scratch: the vertex-key sort and the
	// joins, the host route's staged columns, and the undirected de-duplication.
	WS_KEY_STATUS = 2, WS_KEY_POS = 16, WS_KEY_SCAN = 17, WS_KEY_SORT_A = 18, WS_KEY_SORT_B = 19, WS_KEY_ROW_A = 20,
	WS_KEY_ROW_B = 21, WS_KEY_EDGE_A = 22, WS_KEY_EDGE_B = 23, WS_KEY_EDGE_C = 24,
	WS_KEY_IN_VKEY = 40, WS_KEY_IN_VVALID = 41, WS_KEY_IN_SKEY = 42, WS_KEY_IN_DKEY = 43, WS_KEY_IN_SVALID = 44,
	WS_KEY_IN_DVALID = 45,
	WS_UKEY_MS = 46, WS_UKEY_MD = 47, WS_UKEY_SORT_A = 48, WS_UKEY_SORT_B = 49, WS_UKEY_IDX_A = 50, WS_UKEY_IDX_B = 51,
	WS_UKEY_AUX = 52, WS_UKEY_R_ROW = 53, WS_UKEY_M_ROW = 54, WS_UKEY_DCNT = 55, WS_UKEY_NULL_MULT = 56,
	WS_UKEY_H_LO = 57, WS_UKEY_H_MULT = 58,
	// shortest_path_count and all_shortest_paths (pgq_allshortest.cu): behind each batch's levels, the path counts
	// sigma [n_ab][L] int64 (with WS_LEVEL, which the driver keeps), the batch counters, the step-ordered in-lists
	// (built once per all_shortest_paths call: sorted keys and in-CSR positions, each with the sort's second buffer),
	// and the per-row results the entry points return: counts and list lengths in WS_AS_COUNT / WS_AS_PATH_LEN, the
	// number of lists in WS_AS_NPATHS (their element counts and offsets are shortestpath's WS_OUT_LENGTHS and
	// WS_OUT_OFFSETS).
	WS_AS_SIGMA = 59, WS_AS_COUNTERS = 60, WS_AS_STEP_KEY_A = 61, WS_AS_STEP_KEY_B = 62, WS_AS_STEP_POS_A = 63,
	WS_AS_STEP_POS_B = 64, WS_AS_COUNT = 65, WS_AS_NPATHS = 66, WS_AS_PATH_LEN = 67,
	// The walk engine (pgq_count.cuh) of shortest_k_paths (pgq_kshortest.cu) and of all_cheapest_paths (pgq_cheapest.cu),
	// which also reads all_shortest_paths' step lists: each lane's row and internal ids; a batch's backward reach (reach,
	// frontier and next-frontier masks [n][W / 64]); its two rolling count layers [n_ab][W], each lane's running total,
	// alive flag and counting bit, the call's counters; per row the walks, their elements, the last walk's length, the
	// first walk and the first element; a storing group's lanes, their sources and its layers; and the walks' offsets,
	// their elements and the scans' total.
	WS_KS_LANE_ROW = 68, WS_KS_PSRC = 69, WS_KS_PDST = 70, WS_KS_REACH = 71, WS_KS_FRONT = 72, WS_KS_NEXT = 73,
	WS_KS_OMEGA_A = 74, WS_KS_OMEGA_B = 75, WS_KS_TOTAL = 76, WS_KS_ALIVE = 77, WS_KS_ACTIVE = 78, WS_KS_COUNTERS = 79,
	WS_KS_NPATHS = 80, WS_KS_ROW_ELEMS = 81, WS_KS_LAST = 82, WS_KS_FIRST = 83, WS_KS_ELEM_OFF = 84,
	WS_KS_GROUP_LANE = 85, WS_KS_GROUP_SRC = 86, WS_KS_LAYERS = 87, WS_KS_WALK_OFF = 88, WS_KS_ELEMS = 89,
	WS_KS_SCAN_TOTAL = 90,
	// shortest_k_paths' path modes (pgq_kpaths_modes.cu), which also read the step lists: the rows' internal ids; a
	// round's spur searches, their ban lists and seed flags; a batch's lane -> spur map, seen / frontier / next masks
	// [n][W / 64], levels [n][W] uint16, done and grew masks, spur lengths and offsets, counters, TRAIL's ban bitmap over
	// out-CSR positions and its (position, lane) table; the spurs' steps and elements.
	WS_KM_IDS = 91, WS_KM_PIDS = 92, WS_KM_SPURS = 93, WS_KM_LISTS = 94, WS_KM_HAS_SEED = 95, WS_KM_LANE_SPUR = 96,
	WS_KM_SEEN = 97, WS_KM_FRONT = 98, WS_KM_NEXT = 99, WS_KM_LEVEL = 100, WS_KM_DONE = 101, WS_KM_GREW = 102,
	WS_KM_HLEN = 103, WS_KM_LANE_OFF = 104, WS_KM_COUNTERS = 105, WS_KM_BAN_BITS = 106, WS_KM_BAN_KEYS = 107,
	WS_KM_STEPS = 108, WS_KM_STEP_ELEMS = 109,
	// shortest_k_groups in WALK mode, on top of shortest_k_paths' slots: each lane's length groups found past h = 0
	WS_KG_GROUPS = 110,
	// cheapest_path_count / all_cheapest_paths (pgq_cheapest.cu), behind the Bellman-Ford sweeps, on top of the walk
	// engine's slots: each step-list entry's parent as an internal id; per lane of a sweep batch its open flag,
	// |B_tight(t)| and infinite flag; per row the count.
	WS_AC_STEP_PAR = 111, WS_AC_OPEN = 115, WS_AC_BSIZE = 119, WS_AC_INF = 124, WS_AC_COUNT = 127,
	// cheapest_k_paths (pgq_cheapest_k.cu), which runs the rounds of the path modes (WS_KM_*: ids, spurs, lists, seed
	// flags, lane map, spur lengths and offsets, TRAIL's ban bitmap and table, steps) over the step lists: a round's
	// root costs; a batch's distances [n][W] as order-preserving keys, dirty bitmap and flags, tight levels [n][W]
	// uint16, banned-vertex masks [n][W / 64], the tight BFS's two vertex frontiers, grew and done masks; the spurs'
	// step weights.
	WS_CK_ROOT = 139, WS_CK_DIST = 140, WS_CK_DIRTY = 141, WS_CK_FLAGS = 142, WS_CK_LEVEL = 143, WS_CK_VBAN = 144,
	WS_CK_FRONT = 145, WS_CK_GREW = 146, WS_CK_DONE = 147, WS_CK_STEP_W = 148,
	// a weighted key build's staged weight column and its validity (with the other WS_KEY_IN_* columns)
	WS_KEY_IN_W = 149, WS_KEY_IN_WVALID = 150,
	WS_SLOTS // (the last block holds the highest numbers)
};

// The rules between the blocks, checked on their names.
constexpr int ws_masks[] = {WS_SEEN, WS_VISIT_A, WS_VISIT_B};
constexpr int ws_radix[] = {WS_RADIX_HIST, WS_RADIX_SCAN};
constexpr int ws_staging[] = {WS_IN_SRC, WS_IN_DST, WS_IN_VALID, WS_OUT_LEN, WS_OUT_VALID, WS_OUT_OFFSETS,
                              WS_IN_DST_VALID, WS_OUT_LENGTHS, WS_OUT_PATH_OFFSETS, WS_OUT_PATH_VALID, WS_AS_COUNT,
                              WS_AS_NPATHS, WS_AS_PATH_LEN};
constexpr int ws_driver[] = {WS_ROW_LANE, WS_STATUS, WS_LEVEL, WS_ITEMS_A, WS_ITEMS_B, WS_TLIST, WS_TBITS, WS_WALK,
                             WS_ELEMS, WS_SLOT_OFF, WS_PSRC, WS_PDST, WS_SATBITS, WS_SHARED_ROWS, WS_LANE_SRC,
                             WS_ASSIGN_TMP, WS_BATCH_ROWS, WS_PATH_TOTAL, WS_SEEN_D, WS_VISIT_A_D, WS_VISIT_B_D,
                             WS_LANE_DST, WS_ITEMS_A_D, WS_ITEMS_B_D, WS_MEET};
constexpr int ws_csr[] = {WS_CSR_SCAN, WS_CSR_ERR, WS_CSR_FLAGS, WS_CSR_WIDE, WS_CSR_EDGE_A, WS_CSR_EDGE_B,
                          WS_CSR_EDGE_C, WS_CSR_VERTEX_A, WS_CSR_VERTEX_B, WS_CSR_VERTEX_C, WS_CSR_VERTEX_D,
                          WS_CSR_VERTEX_E};
constexpr int ws_bf[] = {WS_BF_DIST, WS_BF_DIRTY, WS_BF_FLAGS};
constexpr int ws_cp[] = {WS_CP_LEVEL, WS_CP_PKEY, WS_CP_FRONTIER, WS_CP_LANE_TGT, WS_CP_COUNTERS, WS_ELEMS,
                         WS_PATH_TOTAL};
constexpr int ws_as[] = {WS_AS_SIGMA, WS_AS_COUNTERS, WS_AS_STEP_KEY_A, WS_AS_STEP_KEY_B, WS_AS_STEP_POS_A,
                         WS_AS_STEP_POS_B};
constexpr int ws_ks[] = {WS_KS_LANE_ROW, WS_KS_PSRC, WS_KS_PDST, WS_KS_REACH, WS_KS_FRONT, WS_KS_NEXT, WS_KS_OMEGA_A,
                         WS_KS_OMEGA_B, WS_KS_TOTAL, WS_KS_ALIVE, WS_KS_ACTIVE, WS_KS_COUNTERS, WS_KS_NPATHS,
                         WS_KS_ROW_ELEMS, WS_KS_LAST, WS_KS_FIRST, WS_KS_ELEM_OFF, WS_KS_GROUP_LANE, WS_KS_GROUP_SRC,
                         WS_KS_LAYERS, WS_KS_WALK_OFF, WS_KS_ELEMS, WS_KS_SCAN_TOTAL};
constexpr int ws_km[] = {WS_KM_IDS, WS_KM_PIDS, WS_KM_SPURS, WS_KM_LISTS, WS_KM_HAS_SEED, WS_KM_LANE_SPUR,
                         WS_KM_SEEN, WS_KM_FRONT, WS_KM_NEXT, WS_KM_LEVEL, WS_KM_DONE, WS_KM_GREW, WS_KM_HLEN,
                         WS_KM_LANE_OFF, WS_KM_COUNTERS, WS_KM_BAN_BITS, WS_KM_BAN_KEYS, WS_KM_STEPS,
                         WS_KM_STEP_ELEMS};
constexpr int ws_kg[] = {WS_KG_GROUPS};
constexpr int ws_ac[] = {WS_AC_STEP_PAR, WS_AC_OPEN, WS_AC_BSIZE, WS_AC_INF, WS_AC_COUNT};
constexpr int ws_ck[] = {WS_CK_ROOT, WS_CK_DIST, WS_CK_DIRTY, WS_CK_FLAGS, WS_CK_LEVEL, WS_CK_VBAN, WS_CK_FRONT,
                         WS_CK_GREW, WS_CK_DONE, WS_CK_STEP_W};
constexpr int ws_analytics[] = {WS_LCC_SRC, WS_LCC_OUT, WS_LCC_OUT_VALID, WS_LCC_BIG_ROWS, WS_LCC_BIG_CNT,
                                WS_LCC_SRC_VALID, WS_LCC_BITMAP, WS_AN_REF_OFF, WS_AN_SCAN, WS_PR_KEY_A, WS_PR_KEY_B,
                                WS_PR_VAL_A, WS_PR_VAL_B, WS_PR_IN_OFF, WS_PR_SCAN, WS_PR_DFLAG, WS_PR_RANK,
                                WS_PR_TEMP, WS_PR_CONTRIB, WS_PR_DANGLING, WS_PR_TOTAL, WS_WCC_EDGES, WS_WCC_EDGES + 5,
                                WS_WCC_COMP, WS_WCC_HOOK, WS_WCC_BEST, WS_WCC_MERGE_POS, WS_WCC_MERGE_A,
                                WS_WCC_MERGE_B, WS_WCC_FLAGS, WS_WCC_SORT_KEY, WS_WCC_SORT_IDX_A, WS_WCC_SORT_IDX_B};
constexpr int ws_keys[] = {WS_KEY_STATUS, WS_KEY_POS, WS_KEY_SCAN, WS_KEY_SORT_A, WS_KEY_SORT_B, WS_KEY_ROW_A,
                           WS_KEY_ROW_B, WS_KEY_EDGE_A, WS_KEY_EDGE_B, WS_KEY_EDGE_C, WS_UKEY_MS, WS_UKEY_MD,
                           WS_UKEY_SORT_A, WS_UKEY_SORT_B, WS_UKEY_IDX_A, WS_UKEY_IDX_B, WS_UKEY_AUX, WS_UKEY_R_ROW,
                           WS_UKEY_M_ROW, WS_UKEY_DCNT, WS_UKEY_NULL_MULT, WS_UKEY_H_LO, WS_UKEY_H_MULT};
constexpr int ws_key_staging[] = {WS_KEY_IN_VKEY, WS_KEY_IN_VVALID, WS_KEY_IN_SKEY, WS_KEY_IN_DKEY, WS_KEY_IN_SVALID,
                                  WS_KEY_IN_DVALID, WS_KEY_IN_W, WS_KEY_IN_WVALID};
template <size_t A, size_t B>
constexpr bool ws_disjoint(const int (&a)[A], const int (&b)[B]) {
	for (int x : a) {
		for (int y : b) {
			if (x == y) {
				return false;
			}
		}
	}
	return true;
}
template <size_t A, size_t... B>
constexpr bool ws_apart(const int (&a)[A], const int (&...b)[B]) {
	return (ws_disjoint(a, b) && ...);
}
static_assert(ws_apart(ws_masks, ws_radix, ws_staging, ws_driver, ws_csr, ws_bf, ws_cp, ws_as, ws_ks, ws_km, ws_kg,
                       ws_ac, ws_ck, ws_analytics, ws_keys, ws_key_staging),
              "only the BFS drivers may write the search masks");
static_assert(ws_apart(ws_staging, ws_driver, ws_bf), "a path entry point's staged columns live while its driver runs");
static_assert(ws_apart(ws_cp, ws_staging, ws_bf), "the tight search runs on the distances and columns of its call");
static_assert(ws_apart(ws_as, ws_staging, ws_driver, ws_radix),
              "path counts and step lists live across the batches of their driver, over the columns of their call");
static_assert(ws_apart(ws_ks, ws_staging, ws_driver, ws_radix, ws_as, ws_bf, ws_cp),
              "the walk search lives across its batches and groups, over the columns of its call and the step lists, and "
              "across the sweep batches of all_cheapest_paths, over their distances");
static_assert(ws_apart(ws_km, ws_staging, ws_driver, ws_radix, ws_as, ws_ks),
              "the spur searches live across their rounds, over the step lists; WALK's own slots stay apart");
static_assert(ws_apart(ws_kg, ws_staging, ws_driver, ws_radix, ws_as, ws_ks),
              "the length groups live across the walk search's batches, beside its own slots");
static_assert(ws_apart(ws_ac, ws_staging, ws_bf, ws_as, ws_ks, ws_kg, ws_cp, ws_radix),
              "the tight walk search lives across the sweep batches, over their distances, the columns of its call and the "
              "step lists, beside the walk engine's slots");
static_assert(ws_apart(ws_ck, ws_staging, ws_bf, ws_km, ws_ks, ws_ac, ws_cp, ws_as, ws_radix),
              "the Bellman-Ford spur searches live across their rounds, beside the rounds' own slots, over the step lists "
              "and the columns of their call; the other searches' slots stay apart");
static_assert(WS_OUT_PATH_OFFSETS < WS_SLOTS && WS_OUT_PATH_VALID < WS_SLOTS, "every slot has a buffer");
static_assert(ws_apart(ws_radix, ws_csr, ws_analytics, ws_keys), "radix_sort_pairs' scratch is apart from its callers'");
static_assert(ws_apart(ws_key_staging, ws_keys, ws_csr, ws_radix), "a key build's staged columns live while it builds");

// Scratch of one path-function call (mask arrays etc.), pooled per context and grown on demand.
struct Workspace {
	pgq_ctx *ctx = nullptr; // the context whose pool it belongs to
	void *buf[WS_SLOTS] = {};
	size_t cap[WS_SLOTS] = {};
	cudaStream_t stream = nullptr; // owned stream for host-pointer calls
	cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
	std::vector<cudaEvent_t> ev_pool; // pairs around expansion kernels
	void *pinned = nullptr;           // small pinned status block
	size_t pinned_cap = 0;
	// The three lane-mask arrays are known to hold zeros from row clean_from on, for the CSR / lane width below
	// (a search only ever writes the rows of vertices WITH in-edges, which the internal numbering puts first):
	// a batch then clears just the first clean_from rows.  Reset whenever the arrays or their user change.
	uint64_t clean_csr_uid = 0;
	int clean_w = 0;
	int64_t clean_from = -1;
	const void *clean_ptr[3] = {nullptr, nullptr, nullptr};
};

struct pgq_ctx {
	int device = 0;
	int sm_count = 132; // H100 SXM; set from the device properties by pgq_ctx_create
	std::mutex mu;
	std::condition_variable cv;
	std::vector<Workspace *> free_ws;
	int live_ws = 0; // workspaces in existence (in use + pooled)
	int max_ws = 8;  // upper bound on them: a workspace holds three lane-mask arrays of the graph's size
	// Device buffers of freed CSRs, by exact size: DuckPGQ rebuilds a CSR of the same shape for every
	// query, so the ~20 cudaMalloc / cudaFree pairs of a CSR are paid once per shape, not once per query.
	std::multimap<size_t, void *> buf_cache;
	size_t buf_cache_bytes = 0;
	size_t buf_cache_limit = (size_t)16 << 30;
};

// Pinned staging ring + stream of one host thread for create_csr_vertex / create_csr_edge chunks:
// a chunk is copied into a pinned slot, sent to the device and narrowed / scattered asynchronously;
// nothing waits per chunk (a slot is waited for only when the ring wraps around onto a busy one).
struct StageRing {
	int device = 0;
	cudaStream_t stream = nullptr;
	char *pinned = nullptr; // nslots x slot_bytes
	char *dev = nullptr;    // nslots x slot_bytes
	size_t slot_bytes = 0;
	int nslots = 0;
	int next = 0;
	std::vector<cudaEvent_t> ev; // slot reusable once its event has completed
	~StageRing();
};

struct pgq_csr {
	pgq_ctx *ctx = nullptr;
	int64_t n = 0;
	int64_t m = 0;
	bool finalized = false;
	DirGraph out;
	DirGraph in;
	PullGraph pull; // the in-edges once more, laid out for the fused bottom-up level
	int64_t *edge_ids = nullptr; // [m] edge rowids in out-CSR order (the CSR position when none were given)
	// Internal vertex numbering: vertices are renumbered so that the ones whose masks are actually
	// gathered (out-degree > 0 and in-degree > 0) come first, then in-only, out-only and isolated
	// vertices, each class in its original order.  All device arrays use internal ids; perm/inv
	// translate at the boundary (pairs in, path vertices / downloaded CSR out).
	int32_t *perm = nullptr; // [n] original id -> internal id
	int32_t *inv = nullptr;  // [n] internal id -> original id
	int64_t n_a = 0;         // vertices with out- and in-edges (the randomly gathered part of the masks)
	int64_t n_ab = 0;        // ... plus vertices with only in-edges: the only ones a BFS level can reach
	uint64_t uid = 0;        // unique per CSR object of the process (workspaces remember whose zeros they hold)
	int64_t device_bytes = 0;
	// incremental build state (create_csr_vertex / create_csr_edge chunks)
	std::mutex mu;
	int32_t *st_cnt = nullptr; // [n] per-vertex counts from create_csr_vertex
	bool have_counts = false;
	bool edge_init = false;
	int64_t edge_size = 0;
	int64_t staged = 0;
	int32_t *st_src = nullptr; // [edge_size]
	int32_t *st_dst = nullptr;
	int64_t *st_eid = nullptr;
	int64_t *st_w = nullptr;   // [edge_size] raw 8-byte weights (create_csr_edge's BIGINT / DOUBLE overloads)
	int *d_err = nullptr;      // device flag: a chunk held an id outside [0, n)
	std::vector<std::shared_ptr<StageRing>> rings; // staging rings that still may hold chunks in flight
	// edge weights in out-CSR position order (CSR::w / CSR::w_double, compressed_sparse_row.hpp:32-40)
	int weight_type = 0; // 0 none, 1 BIGINT, 2 DOUBLE
	int64_t *w_bits = nullptr;
	bool neg_weights = false; // some weight is below zero (a NaN is not): cheapest_path_length relaxes from every vertex
	std::unordered_map<void *, size_t> allocs; // every device buffer of this CSR with its size (buffer cache)
	// pagerank / weakly_connected_component of all n + 2 entries, computed on the first call under `mu` and kept
	// on the host (pgq_analytics.cu); pgq_csr_clone does not copy them
	bool pr_done = false;
	int64_t pr_iters = 0;
	std::vector<double> pr_rank;
	bool wcc_done = false;
	std::vector<int64_t> wcc_label;
};

// ---- helpers implemented in pgq_csr.cu ---------------------------------------------------------
int pgq_ws_acquire(pgq_ctx *ctx, Workspace **out);     // blocks while the context's workspace budget is used up
int pgq_ws_try_acquire(pgq_ctx *ctx, Workspace **out); // PGQ_ERR_OOM instead of blocking
int pgq_ws_grow(Workspace *ws, WsSlot slot, size_t bytes, size_t keep_bytes, cudaStream_t s, void **out);
void pgq_ws_release(pgq_ctx *ctx, Workspace *ws);
int pgq_ws_reserve(Workspace *ws, WsSlot slot, size_t bytes, void **out);
// copies a host column (NULL = absent: *dev = NULL) into the slot on the workspace stream
int stage_column(Workspace *ws, WsSlot slot, const void *host, size_t bytes, const void **dev);
int pgq_ws_pinned(Workspace *ws, size_t bytes, void **out);
int pgq_scan_exclusive_i32(const int32_t *in, int32_t *out, int64_t count, int32_t *block_tmp, cudaStream_t s);
size_t pgq_scan_tmp_elems(int64_t count);
// stable LSD radix sort of (int32 or uint64 key, int32 value) pairs by the low end_bit bits; uses WS_RADIX_HIST and
// WS_RADIX_SCAN
int radix_sort_pairs(Workspace *ws, int32_t *keys_a, int32_t *keys_b, int32_t *vals_a, int32_t *vals_b, int64_t count,
                     int end_bit, cudaStream_t s, int32_t **keys_res, int32_t **vals_res);
int radix_sort_pairs(Workspace *ws, uint64_t *keys_a, uint64_t *keys_b, int32_t *vals_a, int32_t *vals_b, int64_t count,
                     int end_bit, cudaStream_t s, uint64_t **keys_res, int32_t **vals_res);

// Holds an acquired workspace (PGQ_TRY(pgq_ws_acquire(ctx, &g.ws))) and releases it on every return.  A call that
// returns before it marked itself settled first waits for what it queued: copies from / to the caller's buffers and
// kernels on the caller's stream must not outlive the call, nor leak into the workspace's next user, nor into the
// buffers a failed build gives back to the cache.
struct WsGuard {
	pgq_ctx *ctx;
	Workspace *ws = nullptr;
	cudaStream_t used = nullptr; // a caller-provided stream the work was enqueued on, if any
	bool has_used = false;
	bool settled = false; // the call has synchronised the workspace stream itself
	explicit WsGuard(pgq_ctx *c) : ctx(c) {
	}
	WsGuard(const WsGuard &) = delete;
	WsGuard &operator=(const WsGuard &) = delete;
	~WsGuard() {
		if (ws) {
			if (!settled) {
				cudaStreamSynchronize(ws->stream);
				if (has_used) {
					cudaStreamSynchronize(used); // kernels queued on the caller's stream still touch the workspace
				}
				cudaGetLastError();
			}
			pgq_ws_release(ctx, ws);
		}
	}
};

// ---- BFS drivers implemented in pgq_bfs.cu -----------------------------------------------------
// One batch of a path-mode BFS call, as the driver hands it to a PathHook behind the batch's last level, while its
// level array is live.  The sources' levels are 0 again (k_path_fix_sources).
struct PathBatch {
	int b0, cnt, L;            // lanes [b0, b0 + cnt) of the call, in a batch L lanes wide
	int levels;                // BFS levels the batch ran
	int64_t rows_ub;           // upper bound of the rows on its lanes (> 0)
	const uint16_t *level;     // [n][L] BFS level of (vertex, lane) in internal ids, 0xFFFF = not reached
	const int32_t *batch_rows; // the batch's rows, *batch_n (device) of them
	const int *batch_n;
	const int32_t *row_lane, *psrc, *pdst; // the call's lane map: lane of each row (-1 = none) and internal ids
	int64_t *out_lengths;      // [p] element count of each row's lists
	int64_t *slot_off;         // [p] each row's slot in the walk buffer (WS_WALK)
	int64_t *walk_bound;       // elements of the walk buffer handed out so far
	Workspace *ws;
	cudaStream_t s;
	pgq_stats *st;
};
// What a path-mode call does with each batch instead of shortestpath's walk.  With `lists` set, the batches leave
// lists in the walk buffer as shortestpath's walk does (a row's element count in out_lengths, its slot in slot_off,
// the buffer grown by the hook), and the driver places them behind the last batch as it places shortestpath's.
struct PathHook {
	bool lists = false;
	virtual int batch(const PathBatch &b) = 0;
};
// shortestpath's list offsets (k_path_offsets, one block): rows [lo, hi) get offsets from `base` on, in row order, from
// their out_lengths (0 = NULL, -1 = [src] -> 1) and out_valid = length > 0; *d_range_total = the rows' element count
void pgq_path_offsets(int64_t base, int64_t lo, int64_t hi, int64_t *out_offsets, int64_t *out_lengths,
                      uint8_t *out_valid, int64_t *d_range_total, cudaStream_t s);
int pgq_bfs_lengths_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                           const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_len,
                           uint8_t *d_out_valid, cudaStream_t stream, pgq_stats *stats);
int pgq_bfs_paths_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                         const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_offsets,
                         int64_t *d_out_lengths, uint8_t *d_out_valid, int64_t **d_out_elems, int64_t *out_total,
                         cudaStream_t stream, pgq_stats *stats);
// shortestpath's BFS (lane assignment, batches, level loop, path mode) with hook->batch in place of the walk
int pgq_bfs_paths_hooked(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                         const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_offsets,
                         int64_t *d_out_lengths, uint8_t *d_out_valid, int64_t **d_out_elems, int64_t *out_total,
                         PathHook *hook, cudaStream_t stream, pgq_stats *stats);
// h_src / h_src_valid: host copies of d_src / d_src_valid (PGQ_OPT_REFERENCE_BATCHING cuts the batches on the host)
int pgq_bfs_reachability_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                                const uint8_t *d_src_valid, const int64_t *h_src, const uint8_t *h_src_valid,
                                const pgq_options *opts, int64_t *d_out_len, uint8_t *d_out_valid, cudaStream_t stream,
                                pgq_stats *stats);
// d_valid: rows whose source AND destination are valid (nullable = all)
int pgq_bfs_bidirectional_device(pgq_csr *csr, Workspace *ws, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                                 const uint8_t *d_valid, const pgq_options *opts, int64_t *d_out_len,
                                 uint8_t *d_out_valid, cudaStream_t stream, pgq_stats *stats);
