/*
 * pgq_oracle_cheapest.c -- CPU restatement of cheapest_path, AN EXTENSION: the reference has no such function.
 *
 * TEST INFRASTRUCTURE ONLY, like pgq_oracle.c: the checker of pgq_cheapest_path.  Only tests/ and tools/ may
 * build, load or call this file; the product never links or falls back to it.
 *
 * The distances are those of cheapest_path_length's batched Bellman-Ford (the sweeps below are pgq_oracle.c's, which
 * tests/test_cheapest_path_edges.py pins to the reference binary), run at a given lane width.  The path is then found
 * by a sequential breadth-first search in the style of shortest_path.cpp:12-41.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_ERR_ALLOC 1
#define ORC_ERR_ARG 2

typedef struct { /* the layout of pgq_oracle.c's orc_stats */
	int64_t batches;
	int64_t levels;
	int64_t edges_traversed;
	int64_t frontier_vertices;
} orc_stats;

/* The sweeps of one batch over dists[v_size][lane_limit]: the loop of pgq_oracle.c's ORC_BF_BODY, restated from
 * TemplatedBatchBellmanFord (cheapest_path_length.cpp:60-71; UpdateOneLane l.29-36). */
#define ORC_BF_SWEEPS(T)                                                                                           \
	int changed = 1;                                                                                               \
	while (changed) { /* l.60-71 */                                                                                \
		changed = 0;                                                                                               \
		for (int64_t vv = 0; vv < v_size; vv++) {                                                                  \
			for (int64_t index = v[vv]; index < v[vv + 1]; index++) {                                              \
				T *vd = dists + vv * lane_limit;                                                                   \
				T *nd = dists + e[index] * lane_limit;                                                             \
				T weight = w[index];                                                                               \
				for (int l = 0; l < lane_limit; l++) { /* UpdateOneLane l.29-36 */                                 \
					T nw = vd[l] + weight;                                                                         \
					if (nw < nd[l]) {                                                                              \
						nd[l] = nw;                                                                                \
						changed = 1;                                                                               \
					}                                                                                              \
				}                                                                                                  \
			}                                                                                                      \
		}                                                                                                          \
	}

/* ------------------------------------------------------------------------------------------
 * cheapest_path -- AN EXTENSION: the reference has no such function.  The weighted form of
 * shortestpath's list: rows take lanes in input order, `lanes` per batch; each batch runs the sweeps
 * above (ORC_BF_SWEEPS) to the distances d, then a breadth-first search per batch over the edges d
 * makes tight for a lane (d(v) + w == d(u) in the weight type's arithmetic, compared as values), in
 * shortest_path.cpp's style (l.12-41): the frontier's vertices in ascending id, their edges in CSR
 * order, and the first parent written kept.  The device picks the same parent with a different
 * formulation (the least (vertex id, adjacency position) key among a level's tight edges into the
 * vertex).  h(s) = 0 and the source is never entered again.  Output as orc_shortestpath's:
 * [src, e1, v1, ..., ek, dst]; NULL for a NULL id, a NULL cost, or a destination the tight edges do
 * not reach; [src] for src == dst.  A batch expands level k while F_k (vertices with h = k in some
 * lane) is not empty and some row with a valid cost and src != dst has not reached its destination.
 * stats: batches; levels = tight levels expanded; frontier_vertices = sum of |F_k|;
 * edges_traversed = their out-edges.  A level beyond 65534 -> ORC_ERR_UNSUPPORTED (the device's
 * levels are uint16).
 * ---------------------------------------------------------------------------------------- */
#define ORC_ERR_UNSUPPORTED 4

static int orc_cmp_i64(const void *a, const void *b) {
	const int64_t x = *(const int64_t *)a, y = *(const int64_t *)b;
	return (x > y) - (x < y);
}

static inline int orc_tight_i64(int64_t dv, int64_t w, int64_t du) {
	return (int64_t)((uint64_t)dv + (uint64_t)w) == du; /* the device's int64 addition wraps */
}
static inline int orc_tight_f64(double dv, double w, double du) {
	return dv + w == du;
}

#define ORC_CHEAPEST_PATH_BODY(T, INF, TIGHT)                                                                      \
	if (lanes <= 0) {                                                                                              \
		return ORC_ERR_ARG;                                                                                        \
	}                                                                                                              \
	orc_stats local;                                                                                               \
	memset(&local, 0, sizeof(local));                                                                              \
	const int lane_limit = lanes;                                                                                  \
	const size_t cells = (size_t)(v_size > 0 ? v_size : 1) * lanes;                                                \
	T *dists = (T *)malloc(cells * sizeof(T));                                                                     \
	int32_t *h = (int32_t *)malloc(cells * sizeof(int32_t));                                                       \
	int64_t *par_v = (int64_t *)malloc(cells * sizeof(int64_t));                                                   \
	int64_t *par_e = (int64_t *)malloc(cells * sizeof(int64_t));                                                   \
	uint8_t *next = (uint8_t *)calloc((size_t)(v_size > 0 ? v_size : 1), 1);                                       \
	int64_t *cur_list = (int64_t *)malloc((size_t)(v_size > 0 ? v_size : 1) * sizeof(int64_t));                    \
	int64_t *next_list = (int64_t *)malloc((size_t)(v_size > 0 ? v_size : 1) * sizeof(int64_t));                   \
	int64_t *tgt = (int64_t *)malloc((size_t)lanes * sizeof(int64_t));                                             \
	size_t cap = 1024, total = 0;                                                                                  \
	int64_t *elems = (int64_t *)malloc(cap * sizeof(int64_t));                                                     \
	int rc = ORC_OK;                                                                                               \
	if (!dists || !h || !par_v || !par_e || !next || !cur_list || !next_list || !tgt || !elems) {                                     \
		rc = ORC_ERR_ALLOC;                                                                                        \
		goto done;                                                                                                 \
	}                                                                                                              \
	for (int64_t b0 = 0; b0 < p; b0 += lanes) {                                                                    \
		const int cnt = (int)(p - b0 < lanes ? p - b0 : lanes);                                                    \
		for (size_t i = 0; i < cells; i++) {                                                                       \
			dists[i] = (INF);                                                                                      \
			h[i] = -1;                                                                                             \
			par_v[i] = -1;                                                                                         \
			par_e[i] = -1;                                                                                         \
		}                                                                                                          \
		for (int l = 0; l < cnt; l++) {                                                                            \
			int64_t row = b0 + l;                                                                                  \
			int sv = !src_valid || src_valid[row], dv = !dst_valid || dst_valid[row];                              \
			if ((sv && (src[row] < 0 || src[row] >= v_size)) || (dv && (dst[row] < 0 || dst[row] >= v_size))) {    \
				rc = ORC_ERR_ARG;                                                                                  \
				goto done;                                                                                         \
			}                                                                                                      \
			if (sv) {                                                                                              \
				dists[src[row] * lanes + l] = 0;                                                                   \
			}                                                                                                      \
		}                                                                                                          \
		local.batches++;                                                                                           \
		{                                                                                                          \
			ORC_BF_SWEEPS(T)                                                                                       \
		}                                                                                                          \
		/* the tight search: F_0 = the sources, the open rows and their targets */                                 \
		int64_t open = 0, nf = 0;                                                                                  \
		for (int l = 0; l < lanes; l++) {                                                                          \
			int64_t row = b0 + l;                                                                                  \
			tgt[l] = -1;                                                                                           \
			if (l >= cnt || (src_valid && !src_valid[row])) {                                                      \
				continue;                                                                                          \
			}                                                                                                      \
			h[src[row] * lanes + l] = 0;                                                                           \
			if (!next[src[row]]) {                                                                                 \
				next[src[row]] = 1;                                                                                \
				cur_list[nf++] = src[row];                                                                         \
			}                                                                                                      \
			if (dst_valid && !dst_valid[row]) {                                                                    \
				continue;                                                                                          \
			}                                                                                                      \
			if (src[row] == dst[row]) {                                                                            \
				tgt[l] = -2;                                                                                       \
			} else if (dists[dst[row] * lanes + l] != (INF)) {                                                     \
				tgt[l] = dst[row];                                                                                 \
				open++;                                                                                            \
			}                                                                                                      \
		}                                                                                                          \
		for (int64_t i = 0; i < nf; i++) {                                                                         \
			next[cur_list[i]] = 0;                                                                                 \
		}                                                                                                          \
		for (int32_t k = 0; nf > 0 && open > 0; k++) {                                                             \
			qsort(cur_list, (size_t)nf, sizeof(int64_t), orc_cmp_i64); /* the frontier in ascending id */          \
			int64_t ne = 0, nn = 0;                                                                                \
			for (int64_t i = 0; i < nf; i++) {                                                                     \
				ne += v[cur_list[i] + 1] - v[cur_list[i]];                                                         \
			}                                                                                                      \
			if (k >= 65534) {                                                                                      \
				rc = ORC_ERR_UNSUPPORTED;                                                                          \
				goto done;                                                                                         \
			}                                                                                                      \
			local.levels++;                                                                                        \
			local.frontier_vertices += nf;                                                                         \
			local.edges_traversed += ne;                                                                           \
			for (int64_t i = 0; i < nf; i++) {                                                                     \
				const int64_t vv = cur_list[i];                                                                    \
				for (int64_t index = v[vv]; index < v[vv + 1]; index++) {                                          \
					int64_t u = e[index];                                                                          \
					for (int l = 0; l < lanes; l++) {                                                              \
						if (h[vv * lanes + l] != k || h[u * lanes + l] != -1 ||                                    \
						    !TIGHT(dists[vv * lanes + l], w[index], dists[u * lanes + l])) {                       \
							continue; /* (a vertex set at this level keeps its first parent) */                    \
						}                                                                                          \
						h[u * lanes + l] = k + 1;                                                                  \
						par_v[u * lanes + l] = vv;                                                                 \
						par_e[u * lanes + l] = index;                                                              \
						if (!next[u]) {                                                                            \
							next[u] = 1;                                                                           \
							next_list[nn++] = u;                                                                   \
						}                                                                                          \
						open -= (u == tgt[l]);                                                                     \
					}                                                                                              \
				}                                                                                                  \
			}                                                                                                      \
			for (int64_t i = 0; i < nn; i++) {                                                                     \
				next[next_list[i]] = 0;                                                                            \
			}                                                                                                      \
			int64_t *t = cur_list;                                                                                 \
			cur_list = next_list;                                                                                  \
			next_list = t;                                                                                         \
			nf = nn;                                                                                               \
		}                                                                                                          \
		for (int l = 0; l < cnt; l++) {                                                                            \
			int64_t row = b0 + l;                                                                                  \
			size_t len = 0;                                                                                        \
			if (tgt[l] == -2) {                                                                                    \
				len = 1;                                                                                           \
			} else if (tgt[l] >= 0 && h[tgt[l] * lanes + l] >= 0) {                                                \
				len = 2 * (size_t)h[tgt[l] * lanes + l] + 1;                                                       \
			}                                                                                                      \
			out_offsets[row] = (int64_t)total;                                                                     \
			out_lengths[row] = (int64_t)len;                                                                       \
			out_valid[row] = len > 0;                                                                              \
			if (total + len > cap) {                                                                               \
				while (total + len > cap) {                                                                        \
					cap *= 2;                                                                                      \
				}                                                                                                  \
				int64_t *e2 = (int64_t *)realloc(elems, cap * sizeof(int64_t));                                   \
				if (!e2) {                                                                                         \
					rc = ORC_ERR_ALLOC;                                                                            \
					goto done;                                                                                     \
				}                                                                                                  \
				elems = e2;                                                                                        \
			}                                                                                                      \
			int64_t *out = elems + total;                                                                          \
			if (len == 1) {                                                                                        \
				out[0] = src[row];                                                                                 \
			} else if (len > 1) {                                                                                  \
				int64_t node = tgt[l];                                                                             \
				for (size_t j = len - 1; j > 0; j -= 2) {                                                          \
					out[j] = node;                                                                                 \
					out[j - 1] = edge_ids[par_e[node * lanes + l]];                                                \
					node = par_v[node * lanes + l];                                                                \
				}                                                                                                  \
				out[0] = node;                                                                                     \
			}                                                                                                      \
			total += len;                                                                                          \
		}                                                                                                          \
	}                                                                                                              \
done:                                                                                                              \
	if (stats) {                                                                                                   \
		*stats = local;                                                                                            \
	}                                                                                                              \
	free(dists);                                                                                                   \
	free(h);                                                                                                       \
	free(par_v);                                                                                                   \
	free(par_e);                                                                                                   \
	free(next);                                                                                                    \
	free(cur_list);                                                                                                \
	free(next_list);                                                                                               \
	free(tgt);                                                                                                     \
	if (rc != ORC_OK) {                                                                                            \
		free(elems);                                                                                               \
		elems = NULL;                                                                                              \
		total = 0;                                                                                                 \
	}                                                                                                              \
	*out_elems = elems;                                                                                            \
	*out_total = (int64_t)total;                                                                                   \
	return rc;

int orc_cheapest_path_i64(int64_t v_size, const int64_t *v, const int64_t *e, const int64_t *edge_ids, const int64_t *w,
                          int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                          const uint8_t *dst_valid, int lanes, int64_t *out_offsets, int64_t *out_lengths,
                          uint8_t *out_valid, int64_t **out_elems, int64_t *out_total, orc_stats *stats) {
	ORC_CHEAPEST_PATH_BODY(int64_t, INT64_MAX / 2, orc_tight_i64)
}

int orc_cheapest_path_f64(int64_t v_size, const int64_t *v, const int64_t *e, const int64_t *edge_ids, const double *w,
                          int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                          const uint8_t *dst_valid, int lanes, int64_t *out_offsets, int64_t *out_lengths,
                          uint8_t *out_valid, int64_t **out_elems, int64_t *out_total, orc_stats *stats) {
	ORC_CHEAPEST_PATH_BODY(double, 1.7976931348623157e308 / 2, orc_tight_f64)
}

void orc_cheapest_free(void *p) {
	free(p);
}
