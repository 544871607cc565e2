/*
 * duckpgq_b200.h -- C ABI of the H100-native (sm_90a) path-finding hot path of DuckPGQ.
 *
 * This is the drop-in boundary: the shared library libduckpgq_b200.so exports exactly these
 * symbols (plain pointers + sizes, caller-owned buffers, int status codes, no C++/torch types,
 * no exception or CUDA error ever crosses it).  Each entry point names the reference interface
 * (cwida/duckpgq-extension @ 8d40274d, paths relative to the reference root) whose work it
 * takes over; INTEGRATION.md shows the DuckDB-side binding for each.
 *
 * Conventions
 *   - vertex ids are the dense rowids [0, n) of the vertex table, edge ids are edge-table rowids
 *     (int64 at the boundary, exactly as DuckDB BIGINT vectors carry them);
 *   - on the device the CSR is int32 (n, m < 2^31 is range-checked -> PGQ_ERR_RANGE);
 *   - validity arrays are one byte per row (1 = valid, 0 = NULL); a NULL pointer = all valid;
 *   - every function returns a pgq_status; pgq_last_error() gives the thread-local message.
 *     The texts for PGQ_ERR_CONSTRAINT / PGQ_ERR_INVALID_ID / PGQ_ERR_NOT_INITIALIZED are the
 *     reference's exception texts so the host shim can rethrow them verbatim.
 */
#ifndef DUCKPGQ_B200_H
#define DUCKPGQ_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PGQ_B200_ABI_VERSION 3

typedef enum pgq_status {
	PGQ_OK = 0,
	PGQ_ERR_INVALID_ARG = 1,     /* null pointer, negative size, bad option */
	PGQ_ERR_CUDA = 2,            /* a CUDA runtime call failed (message has the CUDA error string) */
	PGQ_ERR_OOM = 3,             /* host or device allocation failed */
	PGQ_ERR_CONSTRAINT = 4,      /* "Non-existent/non-unique vertices detected..." csr_creation.cpp:121-125 */
	PGQ_ERR_RANGE = 5,           /* id outside [0,n) or n/m >= 2^31 (the reference has UB here) */
	PGQ_ERR_INVALID_ID = 6,      /* "Invalid ID" iterativelength.cpp:41-43 */
	PGQ_ERR_NOT_INITIALIZED = 7, /* "Need to initialize CSR before doing shortest path" iterativelength.cpp:44-51 */
	PGQ_ERR_UNSUPPORTED = 8      /* e.g. BFS depth beyond the path-mode level counter */
} pgq_status;

typedef struct pgq_ctx pgq_ctx; /* one per (process, device): streams, workspaces, CSR registry */
typedef struct pgq_csr pgq_csr; /* one device-resident CSR (replaces class CSR, compressed_sparse_row.hpp:25-47) */

/* Traversal options.  Zero-initialise for the defaults. */
typedef struct pgq_options {
	int32_t lanes;     /* searches per batch: 64, 128, 256 or 512 (reference: LANE_LIMIT 512,
	                      duckpgq_utils.hpp:10).  0 = pick by graph size.  Results never depend on it. */
	int32_t direction; /* 0 = direction-optimising, 1 = top-down (push) only, 2 = bottom-up (pull) only */
	int32_t alpha;     /* switch to pull when frontier_out_edges * alpha > m.  0 = default (5) */
	int32_t flags;     /* PGQ_OPT_* bits */
	/* Multi-GPU: with shard_count > 1 the call runs only the searches whose ordinal (in lane-assignment
	 * order, after the NULL / src == dst / degree shortcuts) is congruent to shard_index modulo
	 * shard_count, and leaves the other searches' rows at (-1, NULL).  Every rank is given ALL pairs and
	 * the CSR replica; the element-wise MAX of the ranks' (length, valid) columns is the full answer --
	 * the one collective of the multi-GPU path.  0 / 0 = no sharding. */
	int32_t shard_index;
	int32_t shard_count;
} pgq_options;

/* By default rows whose answer follows from the degrees alone take no lane: a source without
 * out-edges or a destination without in-edges is unreachable (NULL), and for shortestpath
 * src == dst is [src].  Results are identical; only the batch composition (and with it the work
 * counters) differs from the reference's, which gives every such row a lane
 * (iterativelength.cpp:93-111).  PGQ_OPT_REFERENCE_BATCHING switches the shortcut off so that
 * batches, levels and edges_traversed equal the reference's for the same lane width. */
#define PGQ_OPT_REFERENCE_BATCHING 1
/* Rows with the SAME source share one search lane by default (the MATCH rewriter emits the cross product
 * of the source and destination sets, match.cpp:476-487: a DataChunk of 2048 rows often holds a handful
 * of distinct sources).  Lanes are numbered by the first appearance of their source, so without repeated
 * sources the composition is the reference's.  The two bits below switch the two shortcuts off
 * individually (PGQ_OPT_REFERENCE_BATCHING switches off both); answers never change. */
#define PGQ_OPT_NO_DEDUP 2
#define PGQ_OPT_NO_PRUNE 4

/* Counters of one path-function call.  edges_traversed is the algorithmic work W of SURVEY.md
 * section 8d: the trip count of the reference's inner loop (iterativelength.cpp:18-24) for the same
 * lane width and batch composition -- it is defined by the frontier sets, not by what the GPU
 * chose to read, and tests check it against the oracle. */
typedef struct pgq_stats {
	int64_t batches;
	int64_t levels;
	int64_t edges_traversed;
	int64_t frontier_vertices;
	int64_t push_levels;
	int64_t pull_levels;
	int64_t kernel_launches; /* CUDA kernels launched by this call */
	int64_t h2d_bytes;
	int64_t d2h_bytes;
	double expand_ms; /* sum of CUDA-event durations of the frontier-expansion kernels */
	double total_ms;  /* CUDA-event duration of the whole call on its stream */
	int32_t lanes;    /* lane width actually used */
	int32_t reserved;
	int64_t searches; /* search lanes run (= distinct sources of the rows that needed a search, unless PGQ_OPT_NO_DEDUP) */
	int64_t pruned;   /* rows answered from the degrees alone (see PGQ_OPT_REFERENCE_BATCHING) */
	int64_t search_rows; /* rows answered by a search lane (>= searches) */
	double pull_ms;      /* the share of expand_ms spent in bottom-up levels (the dominant kernel) ... */
	int64_t pull_edges;  /* ... and the share of edges_traversed those levels account for */
} pgq_stats;

/* ---- library / context --------------------------------------------------------------------- */
int pgq_abi_version(void);
const char *pgq_last_error(void); /* thread-local, valid until the next call on this thread */
const char *pgq_status_text(int status); /* the reference's exception text for a status, or a generic one */
int pgq_device_count(int *count);
int pgq_ctx_create(int device, pgq_ctx **out);
void pgq_ctx_destroy(pgq_ctx *ctx);

/* ---- CSR lifecycle --------------------------------------------------------------------------
 * The incremental form mirrors the three UDF steps of csr_creation.cpp one to one, so a DuckDB
 * shim can forward every DataChunk as it arrives (the calls are thread-safe: create_csr_edge is
 * invoked concurrently by DuckDB's worker threads, csr_creation.cpp:134 uses an atomic ticket):
 *
 *   pgq_csr_create           <- CsrInitializeVertex          csr_creation.cpp:14-41
 *   pgq_csr_add_vertex_counts<- CreateCsrVertexFunction      csr_creation.cpp:86-110  (v[dense_id+2] = cnt)
 *   pgq_csr_add_edges        <- CreateCsrEdgeFunction        csr_creation.cpp:112-198 (+ CsrInitializeEdge :43-61)
 *   pgq_csr_finalize         <- (implicit in the reference: the CSR is complete when the CTE is drained)
 *   pgq_csr_free             <- DeleteCsrFunction csr_deletion.cpp:10-20 / DuckPGQState::QueryEnd duckpgq_state.cpp:162-170
 *
 * Within one source vertex, edges keep the order in which they were handed to pgq_csr_add_edges
 * (chunk call order, then row order) -- the order a single-threaded reference produces.
 * The chunk calls are ASYNCHRONOUS: a chunk is copied into a pinned staging slot of the calling thread
 * and travels to the device behind the call's back; an id outside [0, n) is therefore reported by
 * pgq_csr_finalize (PGQ_ERR_RANGE), not by the chunk call that carried it.
 */
int pgq_csr_create(pgq_ctx *ctx, int64_t n_vertices, pgq_csr **out);
int pgq_csr_add_vertex_counts(pgq_csr *csr, int64_t count, const int64_t *dense_id, const int64_t *cnt,
                              int64_t *sum_out /* nullable: += sum(cnt) of this chunk */);
int pgq_csr_add_edges(pgq_csr *csr, int64_t edge_size /* arg 2: sum of cnt */,
                      int64_t edge_size_count /* arg 3: count(*) of the edge join */, int64_t count,
                      const int64_t *src_rowid, const int64_t *dst_rowid, const int64_t *edge_rowid);
/* The BIGINT / DOUBLE weight overloads of create_csr_edge (csr_creation.cpp:141-198,227-235): as
 * pgq_csr_add_edges plus one weight per row (CSR::w / CSR::w_double, compressed_sparse_row.hpp:32-40);
 * exactly one of weight_i64 / weight_f64 is given, the same one for every chunk of a CSR. */
int pgq_csr_add_edges_weighted(pgq_csr *csr, int64_t edge_size, int64_t edge_size_count, int64_t count,
                               const int64_t *src_rowid, const int64_t *dst_rowid, const int64_t *edge_rowid,
                               const int64_t *weight_i64, const double *weight_f64);
int pgq_csr_finalize(pgq_csr *csr);
void pgq_csr_free(pgq_csr *csr);

/* Bulk forms.  pgq_csr_build = the whole CSR CTE (compressed_sparse_row.cpp:234-251) for host
 * columns (src, dst, edge rowid): degree histogram -> prefix sum -> stable scatter, all on the
 * device.  pgq_csr_upload takes a finished host CSR in the reference's own layout
 * (v has n+2 entries with v[i]..v[i+1] the adjacency of i; int64 everywhere) -- what a shim does
 * when the reference's create_csr_* already ran on the CPU.  edge_ids may be NULL (then
 * pgq_shortestpath reports CSR offsets as edge ids). */
int pgq_csr_build(pgq_ctx *ctx, int64_t n_vertices, int64_t n_edges, const int64_t *src_rowid,
                  const int64_t *dst_rowid, const int64_t *edge_rowid, pgq_csr **out);
int pgq_csr_upload(pgq_ctx *ctx, int64_t n_vertices, int64_t n_edges, const int64_t *v, const int64_t *e,
                   const int64_t *edge_ids, pgq_csr **out);
/* pgq_csr_build for edge columns that already live in HBM on the context's device (e.g. handed over
 * by an Arrow / cuDF scan): int32 vertex rowids, int64 edge rowids (NULL = 0..m-1).  The inputs are
 * not modified.  They may still be in the making on any stream of the caller: the call waits for the device
 * (cudaDeviceSynchronize) before it reads them. */
int pgq_csr_build_device(pgq_ctx *ctx, int64_t n_vertices, int64_t n_edges, const int32_t *d_src_rowid,
                         const int32_t *d_dst_rowid, const int64_t *d_edge_rowid, pgq_csr **out);
/* The whole directed CSR CTE (CreateDirectedCSRCTE, compressed_sparse_row.cpp:132-143,234-251) from the columns a
 * user holds: the vertex table's BIGINT key column (its rowid = the position) and the edge table's BIGINT src / dst
 * key columns (its rowid = the position).  A NULL key (validity byte 0) matches nothing.  With ms(k) / md(k) the
 * number of vertex rows whose key equals edge k's src / dst, the CTE gives vertex row a the degree
 * count(k.src) of v a LEFT JOIN e k ON k.src = a.id (S = sum ms in all) and hands create_csr_edge the
 * C = sum ms * md rows (a.rowid, c.rowid, k.rowid) of e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst.
 *   - S != C, or any edge with ms >= 1 and md != 1 -> PGQ_ERR_CONSTRAINT (the text of csr_creation.cpp:121-125;
 *     the reference throws on S != C only and scatters out of place when a dangling dst balances a duplicated one);
 *   - a duplicated source key is legal: the edge is in the adjacency of every matching source row;
 *   - within a source row, edges are in ascending edge rowid order (the order pgq_csr_build gives the same rows);
 *   - n_vertices, n_edges and C must be < 2^31 -> PGQ_ERR_RANGE.
 * The key -> rowid join runs on the device; only a small status block comes back before the rows go through
 * pgq_csr_build_device's pipeline. */
int pgq_csr_build_keys(pgq_ctx *ctx, int64_t n_vertices, const int64_t *vertex_keys, const uint8_t *vertex_key_valid,
                       int64_t n_edges, const int64_t *edge_src_keys, const int64_t *edge_dst_keys,
                       const uint8_t *edge_src_valid, const uint8_t *edge_dst_valid, pgq_csr **out);
/* pgq_csr_build_keys for columns that already live in HBM on the context's device.  The inputs are not modified.
 * As for pgq_csr_build_device, they may still be in the making on any stream of the caller: the call waits for
 * the device (cudaDeviceSynchronize) before it reads them. */
int pgq_csr_build_keys_device(pgq_ctx *ctx, int64_t n_vertices, const int64_t *d_vertex_keys,
                              const uint8_t *d_vertex_key_valid, int64_t n_edges, const int64_t *d_edge_src_keys,
                              const int64_t *d_edge_dst_keys, const uint8_t *d_edge_src_valid,
                              const uint8_t *d_edge_dst_valid, pgq_csr **out);
/* The undirected CSR CTE (CreateUndirectedCSRCTE, compressed_sparse_row.cpp:125-130,145-172,192-223; emitted for
 * every undirected MATCH and for the weakly_connected_component / local_clustering_coefficient table functions) from
 * the same columns as pgq_csr_build_keys.  A NULL key (validity byte 0) matches nothing.
 *   - edges_cte = every (a, c, k) with vertex row a holding key e.src[k] and row c holding e.dst[k]; the CSR rows are
 *     the distinct pairs (p, q) of edges_cte and its reverse (c, a, k), R in all: parallel edges collapse, a -> b and
 *     b -> a give one row each way, a self-loop stays once;
 *   - the degree of row a = the number of distinct "other end" values over the edges incident to a's key in either
 *     direction (the UNION BY NAME of the two join branches grouped by rowid), a NULL or unmatched other end
 *     included; S = their sum;
 *   - S != R -> PGQ_ERR_CONSTRAINT (the text of csr_creation.cpp:121-125), and so is S == R with some row whose R(p)
 *     differs from its degree (the reference scatters out of place there).  A dangling end balanced by a duplicated
 *     key can give R(p) == degree(p) for every row: that CSR is well-formed and is built;
 *   - two choices the reference leaves open (any_value, hash order) are defined: a pair's edge id is the SMALLEST edge
 *     rowid of its group (both directions), and within a row the neighbours are in ascending rowid order;
 *   - an edge table that joins to no pair gives the reference no CSR at all (create_csr_edge never runs); here, as for
 *     pgq_csr_build_keys, it gives the edgeless CSR of n_vertices rows when S == 0 and PGQ_ERR_CONSTRAINT otherwise;
 *   - n_vertices, n_edges and the 2 * sum ms * md rows before de-duplication must be < 2^31 -> PGQ_ERR_RANGE, checked
 *     before they are allocated. */
int pgq_csr_build_keys_undirected(pgq_ctx *ctx, int64_t n_vertices, const int64_t *vertex_keys,
                                  const uint8_t *vertex_key_valid, int64_t n_edges, const int64_t *edge_src_keys,
                                  const int64_t *edge_dst_keys, const uint8_t *edge_src_valid,
                                  const uint8_t *edge_dst_valid, pgq_csr **out);
/* pgq_csr_build_keys_undirected for columns that already live in HBM on the context's device, with the contract of
 * pgq_csr_build_keys_device (inputs not modified; the call waits for the device before it reads them). */
int pgq_csr_build_keys_undirected_device(pgq_ctx *ctx, int64_t n_vertices, const int64_t *d_vertex_keys,
                                         const uint8_t *d_vertex_key_valid, int64_t n_edges,
                                         const int64_t *d_edge_src_keys, const int64_t *d_edge_dst_keys,
                                         const uint8_t *d_edge_src_valid, const uint8_t *d_edge_dst_valid,
                                         pgq_csr **out);
/* The weighted one-shot builds: the same inputs, checks and results as the unweighted entry point each one names, plus
 * the weight column of the 8-argument create_csr_edge (csr_creation.cpp:141-198,227-235), in the form of
 * pgq_csr_add_edges_weighted: exactly one of the *_i64 (BIGINT) / *_f64 (DOUBLE) pointers, else PGQ_ERR_INVALID_ARG.
 * The pointer names the weight type even when there are no edges, so it must be given for n_edges = 0 as well (it is
 * not read then), and such a CSR reports that type -- unlike a chunked build that never received a row, which stays
 * at type 0.  The cheapest functions answer on an edgeless weighted CSR as on any weighted graph without the path.
 *   - positions: the weight of a CSR position is the weight of the input row that became that position.  For the
 *     rows forms that is the order pgq_csr_build gives (stable by source); pgq_csr_upload_weighted takes one weight
 *     per CSR position (the reference's CSR::w / CSR::w_double, compressed_sparse_row.hpp:32-40).  In the key forms
 *     edge k becomes ms(k) rows, one per matching source row, and every one of them carries w[k], as the CTE's join
 *     hands k.w to create_csr_edge on every joined row;
 *   - bits: BIGINT and DOUBLE weights are copied as 8-byte patterns (NaN payloads and -0.0 survive);
 *     pgq_csr_weight_type answers 1 or 2 and pgq_csr_download_weights returns the column in CSR position order;
 *   - NULL weights (the key forms only; weight_valid nullable = all valid): an edge that joins (gives at least one
 *     row) with a NULL weight -> PGQ_ERR_INVALID_ARG, the message names its edge row.  An edge that joins nothing may
 *     have a NULL weight: its row never reaches create_csr_edge.  (The reference skips a NULL-weight row and leaves a
 *     malformed CSR; DESIGN.md section 7.)  The check runs on the device beside the join's own;
 *   - there is no weighted form of pgq_csr_build_keys_undirected: the reference's undirected CTE carries no weights,
 *     and its de-duplication of (p, q) pairs would have to pick one weight out of several. */
int pgq_csr_build_weighted(pgq_ctx *ctx, int64_t n_vertices, int64_t n_edges, const int64_t *src_rowid,
                           const int64_t *dst_rowid, const int64_t *edge_rowid, const int64_t *weight_i64,
                           const double *weight_f64, pgq_csr **out);
int pgq_csr_build_device_weighted(pgq_ctx *ctx, int64_t n_vertices, int64_t n_edges, const int32_t *d_src_rowid,
                                  const int32_t *d_dst_rowid, const int64_t *d_edge_rowid,
                                  const int64_t *d_weight_i64, const double *d_weight_f64, pgq_csr **out);
int pgq_csr_upload_weighted(pgq_ctx *ctx, int64_t n_vertices, int64_t n_edges, const int64_t *v, const int64_t *e,
                            const int64_t *edge_ids, const int64_t *w_i64, const double *w_f64, pgq_csr **out);
int pgq_csr_build_keys_weighted(pgq_ctx *ctx, int64_t n_vertices, const int64_t *vertex_keys,
                                const uint8_t *vertex_key_valid, int64_t n_edges, const int64_t *edge_src_keys,
                                const int64_t *edge_dst_keys, const uint8_t *edge_src_valid,
                                const uint8_t *edge_dst_valid, const int64_t *weight_i64, const double *weight_f64,
                                const uint8_t *weight_valid, pgq_csr **out);
int pgq_csr_build_keys_weighted_device(pgq_ctx *ctx, int64_t n_vertices, const int64_t *d_vertex_keys,
                                       const uint8_t *d_vertex_key_valid, int64_t n_edges,
                                       const int64_t *d_edge_src_keys, const int64_t *d_edge_dst_keys,
                                       const uint8_t *d_edge_src_valid, const uint8_t *d_edge_dst_valid,
                                       const int64_t *d_weight_i64, const double *d_weight_f64,
                                       const uint8_t *d_weight_valid, pgq_csr **out);
/* get_csr_v / get_csr_e (src/core/functions/table/pgq_scan.cpp:84-111): copy the CSR back in the
 * reference's layout.  Any output pointer may be NULL. */
int pgq_csr_download(pgq_csr *csr, int64_t *v_out /* n+2 */, int64_t *e_out /* m */, int64_t *edge_ids_out /* m */);
int pgq_csr_info(pgq_csr *csr, int64_t *n_vertices, int64_t *n_edges, int64_t *device_bytes);
/* csr_get_w_type (csr_get_w_type.cpp:13-36): 0 = no weights, 1 = BIGINT, 2 = DOUBLE; and the weights in
 * the reference's CSR position order (get_csr_w, pgq_scan.cpp:113-141) as raw 8-byte values. */
int pgq_csr_weight_type(pgq_csr *csr, int *weight_type);
int pgq_csr_download_weights(pgq_csr *csr, void *w_out /* m x 8 bytes */);

/* ---- path functions -------------------------------------------------------------------------
 * pgq_iterativelength <- IterativeLengthFunction iterativelength.cpp:34-143
 *   out_len[i] = hop count, out_valid[i] = 1; or out_len[i] = -1, out_valid[i] = 0 when the source
 *   is NULL or dst is unreachable; src == dst -> 0 without a search.
 * pgq_shortestpath    <- ShortestPathFunction shortest_path.cpp:43-207
 *   row i's path [src, e1, v1, ..., ek, dst] is out_elems[out_offsets[i] .. +out_lengths[i]);
 *   out_valid[i] = 0 for NULL.  *out_elems is allocated by the library: release with pgq_free().
 *   Tie-break = the reference's: parent = smallest frontier vertex with an edge to the node,
 *   edge = first matching edge in that vertex's adjacency.
 * Host pointers in, host pointers out; pairs go H2D and results D2H inside the call.
 */
int pgq_iterativelength(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                        const uint8_t *src_valid, const pgq_options *opts, int64_t *out_len, uint8_t *out_valid,
                        pgq_stats *stats);
int pgq_shortestpath(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                     const uint8_t *src_valid, const pgq_options *opts, int64_t *out_offsets, int64_t *out_lengths,
                     uint8_t *out_valid, int64_t **out_elems, int64_t *out_total, pgq_stats *stats);
void pgq_free(void *p);

/* pgq_iterativelength_bidirectional <- IterativeLengthBidirectionalFunction iterativelength_bidirectional.cpp:43-153
 *   Rows in input order; every row with a valid source, a valid destination and src != dst takes a lane, 512 lanes
 *   per batch, no de-duplication and no degree shortcut.  Each lane searches from src (side 0) and from dst (side 1),
 *   BOTH along out-edges; iteration i = 0, 1, ... runs one BFS level of side i & 1.  out_len[i] = i + 1 for the first
 *   iteration after which the two sides' seen sets share a vertex, out_valid[i] = 1.  A batch ends when every lane
 *   has met, or at the first iteration that adds no bit for any lane of the batch: its lanes not met yet are NULL
 *   (out_len -1, out_valid 0).  Met lanes keep expanding, so a row's answer depends on the rows of its batch.
 *   On a graph holding both directions of every edge the result equals pgq_iterativelength's.
 *   src == dst -> 0 without a lane; a NULL source or a NULL destination (src_valid / dst_valid, nullable) -> NULL
 *   without a lane.  Ids outside [0, n) -> PGQ_ERR_RANGE.
 *   opts (nullable): lanes 0 or 512 (else PGQ_ERR_INVALID_ARG), direction and alpha as for pgq_iterativelength;
 *   flags != 0 or shard_count > 1 -> PGQ_ERR_UNSUPPORTED.  stats: batches, levels (= iterations, both sides) and
 *   edges_traversed (out-edges of the expanded frontiers of both sides) are the reference's. */
int pgq_iterativelength_bidirectional(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                                      const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                                      int64_t *out_len, uint8_t *out_valid, pgq_stats *stats);

/* pgq_reachability <- ReachabilityFunction reachability.cpp:165-254
 *   out[i] = 1 when dst[i] is reachable from src[i] along out-edges (src == dst included), else 0; out_valid[i] = 1.
 *   A NULL source or a NULL destination (src_valid / dst_valid, nullable) gives NULL (out 0, out_valid 0).  Any
 *   non-NULL id outside [0, n) -> PGQ_ERR_RANGE.
 *   By default the rows run exactly as pgq_iterativelength runs them, a NULL destination counting as a NULL source
 *   (de-duplication, degree shortcut, early stop once every row is answered; PGQ_OPT_NO_DEDUP / _NO_PRUNE apply), and
 *   stats equal pgq_iterativelength's.
 *   PGQ_OPT_REFERENCE_BATCHING: the reference's batches.  Rows in input order; a row whose source is new to the batch
 *   opens the next lane, a row whose source is not shares its lane (src == dst rows and rows with a NULL destination
 *   too); a NULL source takes no lane; a batch ends behind the row that opened lane 512.  Every source is seen from the
 *   start and a batch runs until a level adds no bit.  batches, levels and edges_traversed are the reference's for
 *   rows without NULL sources; with them, the reference restarts its next batch early (DESIGN.md section 7), this
 *   call does not.  lanes must be 0 or 512 (else PGQ_ERR_INVALID_ARG).
 *   opts (nullable): direction and alpha as for pgq_iterativelength; shard_count > 1 -> PGQ_ERR_UNSUPPORTED. */
int pgq_reachability(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                     const uint8_t *dst_valid, const pgq_options *opts, uint8_t *out, uint8_t *out_valid,
                     pgq_stats *stats);

/* pgq_cheapest_path_length <- CheapestPathLengthFunction cheapest_path_length.cpp:138-160 (batched
 * Bellman-Ford, TemplatedBatchBellmanFord l.52-105) over a CSR built with pgq_csr_add_edges_weighted.
 *   out_cost[i] = cost of the cheapest path src[i] -> dst[i] as a raw 8-byte value of the CSR's weight type
 *   (int64 for BIGINT weights, double for DOUBLE weights; pgq_csr_weight_type tells which), out_valid[i] = 1;
 *   out_valid[i] = 0 (NULL) when no path exists or the target is NULL (l.90-101).
 * A NULL source gives a NULL result (in the reference it shifts the lanes of all later rows of its batch,
 * l.18-25 vs l.88-93 -- a defect, not a behaviour; see DESIGN.md section 7).  Costs are the least fixed point
 * of the relaxation and therefore bit-identical to the reference's, for doubles too. */
int pgq_cheapest_path_length(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                             const uint8_t *src_valid, const uint8_t *dst_valid, void *out_cost, uint8_t *out_valid,
                             pgq_stats *stats);

/* pgq_cheapest_path: the cheapest path itself, as pgq_shortestpath's list [src, e1, v1, ..., ek, dst] (vertex rowids,
 * edge rowids), over a CSR built with pgq_csr_add_edges_weighted.  No reference function: it is the weighted form of
 * shortestpath (SQL/PGQ's ANY CHEAPEST).
 *   Rows take lanes and batches exactly as in pgq_cheapest_path_length, whose distances d the call computes first.
 *   An edge v -> u is tight for a row when d(v) + w == d(u) in the weight type's arithmetic (int64 addition; double
 *   addition rounded to nearest, compared as values: -0.0 == 0.0, a NaN equals nothing).  The path is shortestpath's
 *   tie-break on the tight edges: fewest edges from src, and walking back from dst, the parent is the smallest vertex
 *   id one level closer to src with a tight edge to the node, and the edge its first tight one in adjacency order.
 *   out_valid[i] = 0 (NULL) when the source or destination is NULL, when pgq_cheapest_path_length's cost is NULL, or
 *   when dst is not reached over tight edges (a valid but meaningless cost at a negative weight, DESIGN.md section 7);
 *   src == dst -> [src].  When d(src) = 0 the path's weights summed from 0, left to right, give the cost bit for bit.
 *   *out_elems is allocated by the library: release with pgq_free().  Errors as pgq_cheapest_path_length's; a tight
 *   path deeper than 65534 edges -> PGQ_ERR_UNSUPPORTED.
 *   stats: batches, levels (Bellman-Ford sweeps) and lanes as pgq_cheapest_path_length's; push_levels (tight levels
 *   expanded), frontier_vertices (sum of their sizes) and edges_traversed (their out-edges). */
int pgq_cheapest_path(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                      const uint8_t *dst_valid, int64_t *out_offsets, int64_t *out_lengths, uint8_t *out_valid,
                      int64_t **out_elems, int64_t *out_total, pgq_stats *stats);

/* pgq_cheapest_path_count / pgq_all_cheapest_paths: every cheapest path of a row (SQL/PGQ's ALL CHEAPEST), over a CSR
 * built with pgq_csr_add_edges_weighted (BIGINT or DOUBLE weights).  No reference function.  For a row (s, t), d is what
 * pgq_cheapest_path_length computes, and an edge v -> u is tight for the row by pgq_cheapest_path's rule: d(v) + w ==
 * d(u) in the weight type's arithmetic (int64 addition; double addition rounded to nearest, compared as values: -0.0 ==
 * 0.0, a NaN equals nothing).
 *   - a cheapest path is a walk [s, e1, v1, ..., eh, t] made only of tight edges, in pgq_shortestpath's format (vertex
 *     rowids; edge rowids from the CSR's edge ids, CSR positions when it was uploaded without ids).  Parallel edges give
 *     distinct paths.  For BIGINT weights with d(s) = 0 and no overflow these are exactly the walks whose weights,
 *     summed from 0, equal the cost.  For DOUBLE weights the tight-edge rule is the contract: with edges 0 -> 1 (0.1),
 *     1 -> 2 (0.2) and 0 -> 2 (0.3), only 0 -> 2 is tight, since 0.1 + 0.2 != 0.3 in double.
 *   - count = the number of such walks, saturated at INT64_MAX, which means "at least INT64_MAX, or infinitely many".  It
 *     is infinite exactly when a cycle of tight edges lies on a tight s -> t walk (a zero-weight self-loop or two-cycle
 *     on a route is enough); a tight cycle that s reaches but that does not reach t changes nothing.  s == t: the count
 *     includes [s] and every closed tight walk through s (1 when every weight is above zero).
 *   - NULL (out_valid 0, count 0, no paths): a NULL source or destination (src_valid / dst_valid, both nullable), a NULL
 *     pgq_cheapest_path_length cost, or no tight walk from s to t: exactly the rows on which pgq_cheapest_path is NULL.
 *   - order: by the number of edges ascending; within one length as pgq_all_shortest_paths orders paths (walking back
 *     from t, a step is (the parent's ORIGINAL id, the edge's position in the parent's adjacency), steps compared
 *     lexicographically from t back to s).  Path 0 is pgq_cheapest_path's path: it has the fewest edges, and at each
 *     remaining length the walk back picks a parent whose depth over tight edges is one less.  With every weight 1
 *     (BIGINT), count and paths equal pgq_shortest_path_count / pgq_all_shortest_paths, order included.
 * pgq_all_cheapest_paths lists the first min(count, max_paths) paths of each row (all of them for max_paths == 0; a row
 * with infinitely many still gets its first max_paths), in pgq_shortest_k_paths' layout: row i's out_npaths[i] paths are
 * the call's paths out_first_path[i] .. + out_npaths[i]; path j is (*out_elems)[(*out_path_offsets)[j] ..
 * (*out_path_offsets)[j + 1]); *out_total_paths paths in all.  Both arrays are allocated by the library (also for zero
 * rows): release them with pgq_free().
 *   - errors: max_paths < 0 -> PGQ_ERR_INVALID_ARG; max_paths == 0 with a count of INT64_MAX -> PGQ_ERR_UNSUPPORTED; an
 *     unweighted, missing or unfinalised CSR and ids outside [0, n) give pgq_cheapest_path's errors; a path the result
 *     needs longer than 65533 edges, or a row still counting after 65533 edges -> PGQ_ERR_UNSUPPORTED (this bounds the
 *     call); a row whose count layers, (H + 1) x n_ab x 8 bytes (H its last listed path's length), exceed the layer
 *     budget (4 GiB) -> PGQ_ERR_UNSUPPORTED; an element total that overflows int64 or cannot be allocated ->
 *     PGQ_ERR_OOM; both checked before anything of that size is allocated.
 *   - the call: rows take lanes and batches exactly as in pgq_cheapest_path_length, whose sweeps run first.  Behind each
 *     batch's sweeps, a BFS back from the lanes' targets over their tight edges finds B(t), the vertices with a tight
 *     walk to t (s outside B(t): NULL); then the tight walks from s inside B(t) are counted layer by layer.  A lane stops
 *     after the layer h where the counts are zero on all of B(t) (the count is exact), where its total saturates, or
 *     once h >= |B(t)| with counts still alive (the count is infinite), but not before it has max_paths paths to list.
 *   - stats: batches, levels (Bellman-Ford sweeps) and lanes as pgq_cheapest_path_length's for the same rows;
 *     push_levels = the sum over batches of the tight backward BFS's levels (1 + the largest tight distance to a lane's
 *     target: the last level adds nothing); pull_levels = the sum over batches of the count layers h >= 1 computed (its
 *     lanes' largest stopping layer); kernel_launches, h2d_bytes, d2h_bytes and total_ms cover the whole call. */
int pgq_cheapest_path_count(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                            const uint8_t *src_valid, const uint8_t *dst_valid, int64_t *out_count, uint8_t *out_valid,
                            pgq_stats *stats);
int pgq_all_cheapest_paths(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                           const uint8_t *src_valid, const uint8_t *dst_valid, int64_t max_paths, int64_t *out_count,
                           int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid, int64_t **out_path_offsets,
                           int64_t **out_elems, int64_t *out_total_paths, pgq_stats *stats);

/* pgq_shortest_path_count / pgq_all_shortest_paths: every shortest path of a row (SQL/PGQ's ALL SHORTEST, which the
 * reference rejects).  No reference function.  For a row (s, t) with h = the BFS depth of t from s along out-edges:
 *   - a shortest path is any list [s, e1, v1, ..., eh, t] of h edges along out-edges, in pgq_shortestpath's format
 *     (vertex rowids; edge rowids from the CSR's edge ids, CSR positions when it was uploaded without ids).  Parallel
 *     edges give distinct paths (so does an edge rowid that a duplicated source key of pgq_csr_build_keys put into
 *     several adjacencies).
 *   - count = the number of such lists = (A^h)[s, t], A the adjacency matrix with edge multiplicities; exact up to
 *     INT64_MAX, which it saturates at ("at least INT64_MAX").  s == t -> count 1, the one path [s].
 *   - NULL (out_valid 0, count 0): a NULL source or destination (src_valid / dst_valid, both nullable), or t not
 *     reachable.  Ids outside [0, n) of a row whose ids are both valid -> PGQ_ERR_RANGE; a missing or unfinalised CSR ->
 *     pgq_shortestpath's errors; a depth beyond path mode's limit (65533) -> PGQ_ERR_UNSUPPORTED.
 *   - the order of the paths: walking back from t, a step is (the parent one level closer to s, the edge's position in
 *     the parent's adjacency as pgq_csr_download returns it), steps compared by the parent's ORIGINAL id first, then by
 *     the position; paths ordered lexicographically by their steps from t back to s.  Path 0 is pgq_shortestpath's.
 *   - opts (nullable): lanes, direction, alpha and flags as for pgq_shortestpath (a flag never changes a result);
 *     shard_count > 1 -> PGQ_ERR_UNSUPPORTED.  The rows run exactly as pgq_shortestpath runs them, a NULL destination
 *     counting as a NULL source; its BFS counters (batches, levels, edges_traversed, frontier_vertices, push_levels,
 *     pull_levels, lanes, searches, pruned, search_rows) are pgq_shortestpath's for the same rows when no destination
 *     is NULL.  kernel_launches and total_ms include the path counts and lists (not the launches inside the step-list
 *     sort of pgq_all_shortest_paths).
 * pgq_all_shortest_paths also returns the paths: row i has out_npaths[i] = min(count, max_paths) lists (all of them for
 * max_paths == 0), the first in the order above, each of out_path_len[i] = 2h + 1 elements, back to back from
 * (*out_elems)[out_offsets[i]] (rows in row order; a NULL row has none).  *out_elems is allocated by the library:
 * release with pgq_free().  max_paths < 0 -> PGQ_ERR_INVALID_ARG; max_paths == 0 with a saturated count ->
 * PGQ_ERR_UNSUPPORTED; an element total that overflows int64 or cannot be allocated -> PGQ_ERR_OOM (checked before it
 * is allocated).  Ranks stay exact when counts saturate: every rank listed is below INT64_MAX. */
int pgq_shortest_path_count(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                            const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                            int64_t *out_count, uint8_t *out_valid, pgq_stats *stats);
int pgq_all_shortest_paths(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                           const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts,
                           int64_t max_paths, int64_t *out_count, int64_t *out_npaths, int64_t *out_path_len,
                           int64_t *out_offsets, uint8_t *out_valid, int64_t **out_elems, int64_t *out_total,
                           pgq_stats *stats);

/* pgq_shortest_k_paths: the k shortest walks of a row (SQL/PGQ's SHORTEST k; the reference parses it and rejects it).
 * No reference function.  SQL/PGQ's default path mode is WALK, and the reference supports no other, so vertices and
 * edges may repeat.  For a row (s, t) and k >= 1:
 *   - a walk of h edges is a list [s, e1, v1, ..., eh, t] in pgq_shortestpath's format (vertex rowids; edge rowids from
 *     the CSR's edge ids, CSR positions when it was uploaded without ids).  Parallel edges give distinct walks.  There
 *     are (A^h)[s, t] walks of h edges, A the adjacency matrix with edge multiplicities.
 *   - order: by h ascending; walks of the same h exactly as pgq_all_shortest_paths orders paths (walking back from t, a
 *     step is (the parent's ORIGINAL id, the edge's position in the parent's adjacency as pgq_csr_download returns
 *     it), steps compared lexicographically from t back to s).
 *   - result: the first min(k, total) walks in that order.  A row gets fewer than k walks only when it has fewer than k
 *     in all, which happens only when no cycle lies on any s -> t walk; then it gets all of them.  s == t: the first
 *     walk is [s] (h = 0), then the closed walks through s.  For k <= count the result equals
 *     pgq_all_shortest_paths(max_paths = k); walk 0 is pgq_shortestpath's path.
 *   - NULL (out_valid 0, no walks): a NULL source or destination (src_valid / dst_valid, both nullable), or t not
 *     reachable from s.
 *   - out_npaths[i] walks of row i are the call's walks out_first_path[i] .. + out_npaths[i]; walk j is
 *     (*out_elems)[(*out_path_offsets)[j] .. (*out_path_offsets)[j + 1]); *out_total_paths walks in all.  Both arrays
 *     are allocated by the library (also for zero rows): release them with pgq_free().
 *   - errors: k < 1 -> PGQ_ERR_INVALID_ARG; opts->lanes not 0 or a multiple of 64 up to 512 -> PGQ_ERR_INVALID_ARG; an
 *     id outside [0, n) in a row whose ids are both valid -> PGQ_ERR_RANGE; a missing or unfinalised CSR ->
 *     pgq_shortestpath's errors; shard_count > 1 -> PGQ_ERR_UNSUPPORTED; a walk the result needs longer than 65533
 *     edges -> PGQ_ERR_UNSUPPORTED (this bounds the call, whatever the graph); a row whose count layers alone,
 *     (H + 1) x n_ab x 8 bytes (H its last walk's length, n_ab the vertices with in-edges), exceed the layer budget
 *     (4 GiB) -> PGQ_ERR_UNSUPPORTED; an element total that overflows int64 or cannot be allocated -> PGQ_ERR_OOM,
 *     checked before anything of that size is allocated.
 *   - counts saturate at INT64_MAX and ranks stay exact anyway: every rank listed is below k.
 *   - the call: the rows whose ids are both valid take lanes in input order (no de-duplication), W per batch (W =
 *     opts->lanes, or for 0 the widest of 512, 256, 128, 64 whose two count layers n_ab x W x 8 bytes fit 4 GiB,
 *     halved while W > 64 and the rows that take lanes are at most W / 2).  A batch finds B(t), the vertices that reach
 *     its lanes' targets (t included), by a BFS back from the targets, then counts the walks layer by layer: a lane
 *     stops after the layer h >= 0 where its running total reaches k or where the walk counts are zero on all of B(t)
 *     (s outside B(t): the row is NULL and its lane stops at layer 0), and a batch runs until all its lanes stop.
 *     Then the rows with walks are regrouped to recompute and keep their layers within the layer budget, and the walks
 *     are unranked.  opts->direction, alpha and flags are not used.
 *   - stats: batches; lanes = W; searches = the rows that took a lane; levels = the sum over batches of the layers
 *     h >= 1 each computed (its lanes' largest stopping layer); push_levels = the sum over batches of the backward
 *     BFS's levels (1 + the largest distance to a lane's target from a vertex that reaches it: the last level adds
 *     nothing); kernel_launches, h2d_bytes, d2h_bytes and total_ms (the whole call).  The other counters are 0. */
int pgq_shortest_k_paths(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                         const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts, int64_t k,
                         int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
                         int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths,
                         pgq_stats *stats);

/* SQL/PGQ's path modes (PGQPathMode's WALK, TRAIL, ACYCLIC, SIMPLE) */
typedef enum { PGQ_PATH_WALK = 0, PGQ_PATH_TRAIL = 1, PGQ_PATH_ACYCLIC = 2, PGQ_PATH_SIMPLE = 3 } pgq_path_mode;

/* pgq_shortest_k_paths_mode: SHORTEST k with a path mode (the reference rejects every mode but WALK).  PGQ_PATH_WALK
 * is pgq_shortest_k_paths itself, bit for bit; any value outside pgq_path_mode -> PGQ_ERR_INVALID_ARG.  For a row
 * (s, t) and k >= 1:
 *   - format and order are pgq_shortest_k_paths': a path is [s, e1, v1, ..., eh, t], paths by h, then by their steps
 *     (the parent's ORIGINAL id, the edge's position in the parent's adjacency) from t back to s.  The result is the
 *     first min(k, total) paths the mode admits in that order, i.e. pgq_shortest_k_paths' walk sequence filtered to
 *     the mode, first k; the total is always finite.
 *   - ACYCLIC: no vertex repeats.  SIMPLE: no vertex repeats except that the first may equal the last (for s != t
 *     exactly ACYCLIC).  TRAIL: no edge repeats, an edge being an adjacency entry (parent, position): parallel edges
 *     are distinct, and on an undirected CSR the two directions of an undirected edge are two entries, so a trail may
 *     go u -> v -> u.  A trail may pass through t and come back to it.
 *   - s == t: ACYCLIC gives [s] alone; SIMPLE gives [s], then the simple cycles through s (a self-loop on s is one);
 *     TRAIL gives [s], then the closed trails through s.
 *   - k = 1 gives pgq_shortestpath's path ([s] when s == t).  When a row has at least k shortest paths, the result is
 *     pgq_all_shortest_paths(max_paths = k) in every mode (except SIMPLE and TRAIL at s == t).
 *   - outputs, NULL rows (out_valid 0: a NULL id, or no path), lanes, PGQ_ERR_RANGE, a missing or unfinalised CSR,
 *     shard_count > 1 and the element-total check (PGQ_ERR_OOM before anything of that size is allocated) are
 *     pgq_shortest_k_paths'.  PGQ_ERR_UNSUPPORTED when a spur search reaches a vertex 65534 edges from its spur node
 *     before its target, or when a row accepts a path longer than 65533 edges.
 *   - the call (DESIGN.md §3): Yen's algorithm with Lawler's rule.  Round 0 runs one search per row with s != t, from
 *     s with no bans (s == t: path 0 is [s] with no search).  Each later round takes, for every row still short of k
 *     paths, the path P it accepted last (L edges, found at spur index dev) and runs a spur search from P[j] for
 *     ACYCLIC, and SIMPLE with s != t, at dev <= j < L; SIMPLE with s == t at j = 0 when P = [s], else dev <= j < L;
 *     TRAIL at dev <= j <= L.  The search is a BFS from u = P[j] whose first edge avoids edge j of every accepted path
 *     that shares P's first j steps; ACYCLIC and SIMPLE ban P[0 .. j] (t exempt for SIMPLE at s == t), TRAIL bans P's
 *     first j edges at every level.  Its path back from t takes the first admissible step in step order.  The new
 *     candidates join the row's pool unless already known, and each row then accepts its pool's least path; a row
 *     stops with k paths or an empty pool.  A round's searches take lanes in (row, j) order, W per batch, batches
 *     never mixing rounds; a search whose spur node has no admissible first edge takes no lane.  W = opts->lanes, or
 *     for 0 the widest of 512 .. 64 whose level array n x W x 2 bytes fits 4 GiB, halved while W > 64 and the round's
 *     searches are at most W / 2.  opts->direction, alpha and flags are not used.
 *   - stats: batches (spur batches over all rounds); lanes (the widest W of the call's rounds, round 0 included);
 *     searches (spur searches that took a lane); levels (the sum over batches of the forward expansions run: a batch
 *     expands while a lane that has not reached its target has a non-empty frontier); kernel_launches, h2d_bytes,
 *     d2h_bytes, total_ms as in pgq_shortest_k_paths.  The other counters are 0. */
int pgq_shortest_k_paths_mode(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                              const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts, int64_t k,
                              int32_t path_mode, int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
                              int64_t **out_path_offsets, int64_t **out_elems, int64_t *out_total_paths,
                              pgq_stats *stats);

/* pgq_cheapest_k_paths: the k cheapest paths of a row in a path mode (SQL/PGQ's CHEAPEST k; no reference function),
 * over a CSR built with pgq_csr_add_edges_weighted (BIGINT or DOUBLE weights).  For a row (s, t), a path mode M (a
 * pgq_path_mode; another value -> PGQ_ERR_INVALID_ARG) and k >= 1:
 *   - weights: every weight must be >= 0 (-0.0 is not below zero); a CSR with a weight below zero (a spur search would
 *     need negative-cycle detection, and the cheapest ACYCLIC path under a negative cycle is NP-hard to find) ->
 *     PGQ_ERR_UNSUPPORTED, checked before any work.  An edge of NaN weight belongs to no path.
 *   - cost(P) = P's weights added left to right from 0 in the weight type's arithmetic (int64 addition; double addition
 *     rounded to nearest).  A list is not a path when its cost is NaN or reaches pgq_cheapest_path_length's sentinel
 *     (INT64_MAX / 2; DBL_MAX / 2), tested before each addition (for BIGINT w < sentinel - c), so nothing overflows.
 *     Prefix costs never decrease, so a row has a path exactly when pgq_cheapest_path_length's cost is not NULL, as
 *     long as every BIGINT weight is at most 2^62.  Above that pgq_cheapest_path_length's sums are the reference's
 *     and are not defined (DESIGN.md §3): they can wrap on a route from s (0 -> 1 -> 2 over weights [1, INT64_MAX]
 *     gets a negative cost there and NULL here) or from a vertex s does not reach, whose sentinel plus the weight
 *     wraps into t (a negative cost there, t's own cheapest path here).
 *   - format, modes and NULL rows are pgq_shortest_k_paths_mode's: a path is [s, e1, v1, ..., eh, t]; WALK, TRAIL,
 *     ACYCLIC and SIMPLE admit paths by the same rules, TRAIL's adjacency-entry edges and the s == t cases included;
 *     NULL (out_valid 0, no paths): a NULL id, or no admitted path.
 *   - order: by cost ascending (compared as values), then by h, then by the steps from t back to s as
 *     pgq_shortest_k_paths orders them.  The result is the first min(k, total) admitted paths in that order; with
 *     weights >= 0 that prefix exists even when zero-cost cycles make WALK's total infinite.  s == t: path 0 is [s]
 *     with cost 0.  With no BIGINT weight above 2^62, k = 1 gives pgq_cheapest_path's path in every mode, with
 *     pgq_cheapest_path_length's cost; with every weight 0 or every weight 1 (BIGINT) the paths are
 *     pgq_shortest_k_paths_mode's.
 *   - DOUBLE: the order above is exact for BIGINT.  For DOUBLE it holds whenever every sum involved is exact (dyadic
 *     weights, for example); when a sum rounds, the construction below is the contract, as the tight-edge rule is for
 *     pgq_all_cheapest_paths.  With edges 0 -> 1 (0.1), 1 -> 2 (0.2) and 0 -> 2 (0.3), WALK's two paths from 0 to 2 are
 *     [0, e, 2] (cost 0.3) and then [0, e, 1, e, 2] (cost 0.1 + 0.2 = 0.30000000000000004).
 *   - outputs: pgq_shortest_k_paths' layout (out_npaths, out_first_path, out_valid, *out_path_offsets, *out_elems,
 *     *out_total_paths), and when out_costs is not null, *out_costs = the *out_total_paths paths' costs as raw 8-byte
 *     values of the weight type.  The arrays are allocated by the library (also for zero rows): release with pgq_free().
 *   - errors: k < 1 -> PGQ_ERR_INVALID_ARG; opts->lanes not 0, 32, 64, 128 or 256 -> PGQ_ERR_INVALID_ARG; an unweighted,
 *     missing or unfinalised CSR -> pgq_cheapest_path's errors; ids outside [0, n) in a row whose ids are both valid ->
 *     PGQ_ERR_RANGE; shard_count > 1 -> PGQ_ERR_UNSUPPORTED; a spur search whose tight depth passes 65534, or a row that
 *     accepts a path longer than 65533 edges -> PGQ_ERR_UNSUPPORTED; an element total that overflows int64 or cannot be
 *     allocated -> PGQ_ERR_OOM, checked before anything of that size is allocated.  opts->direction, alpha and flags
 *     are not used, and no result depends on the lane width.
 *   - the call (DESIGN.md §3): pgq_shortest_k_paths_mode's rounds (Yen's algorithm with Lawler's rule, its spur ranges,
 *     bans, D and pool) with the pool keyed by (cost, h, steps), and WALK spurring at dev <= j <= L like TRAIL, with no
 *     bans beyond D.  A spur search from u = P[j] with root R is a lane of a batched Bellman-Ford: each admissible first
 *     edge u -> x seeds d(x) = min(cost(R) + w); sweeps relax the lane's unbanned edges to the fixed point; a BFS over
 *     the lane's tight edges (d(v) + w == d(x) as values, pgq_cheapest_path's rule) from the tight seeds levels the
 *     vertices; and the walk back from t takes, at level >= 2, the first step-list entry whose parent has level - 1 and
 *     whose edge is tight and not banned, at level 1 the first admissible tight position of u's adjacency.  A spur with
 *     no admissible seed takes no lane.  W = opts->lanes, or for 0 the widest of 256, 128, 64, 32 whose distance array
 *     n x W x 8 bytes fits 2 GiB, halved while W > 32 and the round's searches are at most W / 2; a round's searches take
 *     lanes in (row, j) order, and batches never mix rounds.
 *   - stats: batches (spur batches over all rounds); lanes (the widest W of the call); searches (spur searches that took
 *     a lane); levels (Bellman-Ford sweeps summed over batches: at least one per batch, otherwise not deterministic);
 *     push_levels (tight-BFS levels summed over batches: a batch expands while a lane that has not levelled its target
 *     grew at the last level); kernel_launches, h2d_bytes, d2h_bytes and total_ms (the whole call).  The other counters
 *     are 0. */
int pgq_cheapest_k_paths(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                         const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts, int64_t k,
                         int32_t path_mode, int64_t *out_npaths, int64_t *out_first_path, uint8_t *out_valid,
                         int64_t **out_path_offsets, int64_t **out_elems, void **out_costs, int64_t *out_total_paths,
                         pgq_stats *stats);

/* pgq_shortest_k_groups: the paths of the k shortest lengths of a row (SQL/PGQ's SHORTEST k GROUP; the reference
 * carries the selector in its AST and rejects it).  No reference function.  For a row (s, t), a path mode M (a
 * pgq_path_mode; another value -> PGQ_ERR_INVALID_ARG) and k >= 1:
 *   - the length groups of the row are the lengths h at which M admits at least one s -> t path, h_1 < h_2 < ....  The
 *     result is every M-path whose length is among h_1 .. h_k.  A row has fewer than k groups only when its lengths
 *     run out (for WALK only when no cycle lies on any s -> t walk).
 *   - equivalence: the result is the first N paths of pgq_shortest_k_paths_mode's sequence, N = the number of M-paths
 *     of length <= h_k (the sequence is sorted by length, and a length with no M-path contributes nothing).  Format
 *     and order are that function's: [s, e1, v1, ..., eh, t], by h, then by step order from t back to s.
 *   - max_paths: a row lists min(N, max_paths) paths, all N for max_paths = 0.  max_paths < 0 -> PGQ_ERR_INVALID_ARG;
 *     WALK with max_paths = 0 and a saturated N -> PGQ_ERR_UNSUPPORTED (pgq_all_shortest_paths' rule).
 *   - per row, besides out_npaths, out_first_path and out_valid (pgq_shortest_k_paths' lists): out_ngroups = the
 *     groups found (at most k); out_last_len = h of the last group found (-1: none); out_complete = 1 when the listed
 *     paths are all N.  When max_paths cuts a row in TRAIL, ACYCLIC or SIMPLE mode, out_ngroups and out_last_len
 *     describe only the groups of the paths listed.  out_count (nullable) = N: for WALK exact and saturated at
 *     INT64_MAX, from the walk counts; for the other modes exact when out_complete, else -1 (counting trails or simple
 *     paths is #P-hard: the call does not enumerate past max_paths).  A NULL row has count 0, no groups, last_len -1
 *     and out_complete 1.
 *   - s == t: group 1 is h = 0, [s]; WALK goes on with the closed walks through s, SIMPLE with the simple cycles
 *     through s, TRAIL with the closed trails through s; ACYCLIC has [s] only.
 *   - k = 1 gives pgq_all_shortest_paths(max_paths) for s != t in every mode (shortest walks are acyclic); for WALK
 *     out_count then equals pgq_shortest_path_count.
 *   - NULL rows, PGQ_ERR_RANGE, a missing or unfinalised CSR, lanes, shard_count > 1 -> PGQ_ERR_UNSUPPORTED, the
 *     65533-edge limit (a group past it -> PGQ_ERR_UNSUPPORTED), the layer budget ((h_k + 1) x n_ab x 8 bytes per row)
 *     and the element-total check (PGQ_ERR_OOM before anything of that size is allocated) are
 *     pgq_shortest_k_paths[_mode]'s.
 *   - the call (DESIGN.md §3).  WALK runs pgq_shortest_k_paths' four phases; only the counting pass's stop rule
 *     differs: after layer h >= 1 a lane whose count at t is non-zero adds a group, and it stops after its k-th group
 *     or after a layer whose counts are zero on all of B(t).  The storing pass and the unranking then run over the
 *     listed paths (a row's rank bound is its listed count).  The other modes run pgq_shortest_k_paths_mode's rounds;
 *     only a row's stop test differs: before it accepts its pool's least path, a row stops when the pool is empty, or
 *     when it has k groups and the least path is longer than h_k (complete), or when it already lists max_paths
 *     paths (max_paths > 0; complete exactly when the pool's least path is not part of the result).  A row that
 *     accepts a path goes on to the next round, which spurs off it (s == t: [s] is accepted without a search, and the
 *     row stops there when k = 1).
 *   - stats: pgq_shortest_k_paths' for WALK, pgq_shortest_k_paths_mode's for the other modes, over the rounds and
 *     layers this call runs. */
int pgq_shortest_k_groups(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                          const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts, int64_t k,
                          int32_t path_mode, int64_t max_paths, int64_t *out_count, int64_t *out_ngroups,
                          int64_t *out_last_len, uint8_t *out_complete, int64_t *out_npaths, int64_t *out_first_path,
                          uint8_t *out_valid, int64_t **out_path_offsets, int64_t **out_elems,
                          int64_t *out_total_paths, pgq_stats *stats);
/* pgq_shortest_k_groups_count: WALK only, the counting pass and nothing after it.  out_count, out_ngroups and
 * out_last_len as pgq_shortest_k_groups' for WALK; out_valid = the row has a walk (N > 0).  Its errors and stats are
 * pgq_shortest_k_groups' up to the end of the counting pass (stats: kernel_launches, bytes and total_ms of this call). */
int pgq_shortest_k_groups_count(pgq_csr *csr, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                                const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts, int64_t k,
                                int64_t *out_count, int64_t *out_ngroups, int64_t *out_last_len, uint8_t *out_valid,
                                pgq_stats *stats);

/* ---- the other consumers of the CSR ------------------------------------------------------------------------
 * Host pointers in and out.  As in the reference, "v_size" is n + 2: the two entries n and n + 1 behind the
 * vertices have no edges and take part where the reference lets them.  Results are bit-identical to the reference's.
 *
 * pgq_local_clustering_coefficient <- LocalClusteringCoefficientFunction local_clustering_coefficient.cpp:41-70
 *   out[i] = (float)count / (k * (k - 1.0f)) with k the out-degree of src[i] and count the entries of its
 *   neighbours' lists (neighbours with multiplicity) that are neighbours of src[i]; 0 when k < 2.  A NULL source
 *   gives NULL.  An id outside [0, n) fails the call with PGQ_ERR_RANGE (the reference reads out of bounds).
 *   Computed per call.  stats: kernel_launches, h2d/d2h bytes, total_ms.
 * pgq_pagerank <- PageRankFunction pagerank.cpp:31-84
 *   out[i] = the rank of entry src[i], valid for src[i] in [0, n + 2); NULL source or any other id -> NULL.
 *   *iterations (nullable) = the iteration count of the computation (the reference's iteration_count).
 * pgq_weakly_connected_component <- WeaklyConnectedComponentFunction weakly_connected_component.cpp:37-104
 *   out[i] = the reference's component id (the root of src[i] in its Link forest) for src[i] in [0, n + 2);
 *   NULL source or any other id -> NULL.
 * PageRank and the component ids are computed for all entries on the first call for a CSR (concurrent first
 * callers wait for it) and answered from a host copy afterwards.  stats of the call that computed them:
 * levels = PageRank iterations / Boruvka rounds, kernel_launches, d2h_bytes, total_ms (device time of the
 * computation) and, for pgq_pagerank, expand_ms = device time of the serial dangling-rank fold over all
 * iterations.  A call answered from the copy reports zeros.
 */
int pgq_local_clustering_coefficient(pgq_csr *csr, int64_t n_rows, const int64_t *src, const uint8_t *src_valid,
                                     float *out, uint8_t *out_valid, pgq_stats *stats);
int pgq_pagerank(pgq_csr *csr, int64_t n_rows, const int64_t *src, const uint8_t *src_valid, double *out,
                 uint8_t *out_valid, int64_t *iterations, pgq_stats *stats);
int pgq_weakly_connected_component(pgq_csr *csr, int64_t n_rows, const int64_t *src, const uint8_t *src_valid,
                                   int64_t *out, uint8_t *out_valid, pgq_stats *stats);

/* Device-resident form of pgq_iterativelength: all pointers are device pointers on the CSR's
 * device, the work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = the legacy
 * default stream) and has completed when the call returns.  Used when the pairs already live in
 * HBM (and by bench.py for the kernel-only throughput). */
int pgq_iterativelength_device(pgq_csr *csr, int64_t n_pairs, const int64_t *d_src, const int64_t *d_dst,
                               const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_len,
                               uint8_t *d_out_valid, void *stream, pgq_stats *stats);

/* ---- several GPUs of one box, one process (SURVEY.md section 8e) ------------------------------------------
 * Every search is independent given a read-only CSR: the CSR is replicated (pgq_csr_clone: peer copies over
 * NVLink from the device that built it) and the search lanes of a call are dealt over the devices
 * (pgq_options.shard_*), one persistent host thread per device; each device's thread writes the rows it
 * answered straight into the caller's result columns.  No collective, no per-level exchange.
 *   pgq_multi_csr_create   devices[0] must be the primary's device; replicas + their contexts are owned by the group
 *   pgq_multi_iterativelength   same contract as pgq_iterativelength; stats (nullable) has one entry per device
 */
typedef struct pgq_multi_csr pgq_multi_csr;
int pgq_csr_clone(pgq_csr *csr, pgq_ctx *target, pgq_csr **out);
int pgq_multi_csr_create(pgq_csr *primary, const int *devices, int n_devices, pgq_multi_csr **out);
int pgq_multi_csr_devices(pgq_multi_csr *mc, int *n_devices);
void pgq_multi_csr_free(pgq_multi_csr *mc);
int pgq_multi_iterativelength(pgq_multi_csr *mc, int64_t n_pairs, const int64_t *src, const int64_t *dst,
                              const uint8_t *src_valid, const pgq_options *opts, int64_t *out_len,
                              uint8_t *out_valid, pgq_stats *stats);

#ifdef __cplusplus
}
#endif
#endif /* DUCKPGQ_B200_H */
