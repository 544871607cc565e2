/*
 * pgq_oracle_kshortest.c -- CPU restatement of shortest_k_paths, AN EXTENSION: the reference parses SHORTEST k and
 * rejects it ("TopK has not been implemented yet").
 *
 * TEST INFRASTRUCTURE ONLY, like pgq_oracle.c: the checker of pgq_shortest_k_paths.  Only tests/ and tools/ may build,
 * load or call this file; the product never links or falls back to it.
 *
 * Written from the definitions in include/duckpgq_b200.h alone, over the reference CSR layout (v offsets, e targets,
 * edge ids, original vertex ids), one row at a time:
 *   - B(t), the vertices that reach t (t included), by a sequential BFS back from t over the in-lists; its depth gives
 *     the row's share of push_levels;
 *   - the layers w_h(u) = the number of h-edge walks s -> u for u in B(t) (0 elsewhere), summed over in-edges with
 *     saturation at INT64_MAX, every layer kept; the row stops after the layer where its running total reaches k or
 *     where w_h is zero on all of B(t);
 *   - the walks of each length h, enumerated by a depth-first search back from t that tries, at a node with j steps
 *     left, its in-edges in step order (the parent's id, then the edge's position in the parent's adjacency) whose
 *     parent has w_{j-1} > 0, until the length's share of the k walks is listed.  The device unranks instead.
 *   - the stats at a given lane width: rows with both ids valid take lanes in input order, `lanes` per batch.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_ERR_ALLOC 1
#define ORC_ERR_ARG 2
#define ORC_ERR_RANGE 3
#define ORC_ERR_UNSUPPORTED 4

#define ORC_WALK_MAX 65533 /* the longest walk a result may hold */

static int64_t sat_add(int64_t a, int64_t b) { /* a, b >= 0 */
	return a > INT64_MAX - b ? INT64_MAX : a + b;
}

typedef struct {
	int64_t *data;
	int64_t size, cap;
} vec;

static int vec_push(vec *x, int64_t val) {
	if (x->size == x->cap) {
		int64_t cap = x->cap ? 2 * x->cap : 1024;
		int64_t *d = (int64_t *)realloc(x->data, (size_t)cap * sizeof(int64_t));
		if (!d) {
			return ORC_ERR_ALLOC;
		}
		x->data = d;
		x->cap = cap;
	}
	x->data[x->size++] = val;
	return ORC_OK;
}

typedef struct {
	int64_t n;
	const int64_t *edge_ids;
	int64_t *in_off, *in_src, *in_idx; /* in-lists in step order */
	int64_t *back, *queue;             /* BFS back from t: depth, -1 = does not reach t */
	int64_t **layer;                   /* layer[h][u] = w_h(u) */
	int64_t nlayers, cap_layers;
	int64_t *path, *cursor;
	vec *elems, *offsets;
} orc_ks;

/* the first `want` walks of h edges s -> t in step order */
static int enumerate(orc_ks *a, int64_t t, int64_t h, int64_t want) {
	const int64_t len = 2 * h + 1;
	int64_t got = 0, k = h;
	a->path[2 * h] = t;
	a->cursor[h] = a->in_off[t];
	while (k <= h && got < want) {
		if (k == 0) {
			if (vec_push(a->offsets, a->elems->size)) {
				return ORC_ERR_ALLOC;
			}
			for (int64_t i = 0; i < len; i++) {
				if (vec_push(a->elems, a->path[i])) {
					return ORC_ERR_ALLOC;
				}
			}
			got++;
			k = 1;
			continue;
		}
		const int64_t u = a->path[2 * k];
		const int64_t *prev = a->layer[k - 1];
		int64_t j = a->cursor[k];
		while (j < a->in_off[u + 1] && prev[a->in_src[j]] == 0) {
			j++;
		}
		if (j == a->in_off[u + 1]) {
			k++;
			continue;
		}
		a->cursor[k] = j + 1;
		const int64_t par = a->in_src[j];
		a->path[2 * k - 1] = a->edge_ids[a->in_idx[j]];
		a->path[2 * k - 2] = par;
		k--;
		a->cursor[k] = a->in_off[par];
	}
	return ORC_OK;
}

static int64_t *new_layer(orc_ks *a) {
	if (a->nlayers == a->cap_layers) {
		int64_t cap = a->cap_layers ? 2 * a->cap_layers : 64;
		int64_t **l = (int64_t **)realloc(a->layer, (size_t)cap * sizeof(int64_t *));
		if (!l) {
			return NULL;
		}
		a->layer = l;
		a->cap_layers = cap;
	}
	int64_t *x = (int64_t *)calloc((size_t)a->n + 1, sizeof(int64_t));
	if (x) {
		a->layer[a->nlayers++] = x;
	}
	return x;
}

static void drop_layers(orc_ks *a) {
	for (int64_t i = 0; i < a->nlayers; i++) {
		free(a->layer[i]);
	}
	a->nlayers = 0;
}

/* one row (s, t): its walks appended to elems / offsets; *np = how many; *stop = the last layer computed (0 when none
 * was); *ecc = the depth of the BFS back from t */
static int one_row(orc_ks *a, int64_t s, int64_t t, int64_t kk, int64_t *np, int64_t *stop, int64_t *ecc) {
	const int64_t n = a->n;
	for (int64_t u = 0; u < n; u++) {
		a->back[u] = -1;
	}
	int64_t head = 0, tail = 0;
	a->back[t] = 0;
	a->queue[tail++] = t;
	*ecc = 0;
	while (head < tail) {
		const int64_t u = a->queue[head++];
		*ecc = a->back[u];
		for (int64_t j = a->in_off[u]; j < a->in_off[u + 1]; j++) {
			const int64_t w = a->in_src[j];
			if (a->back[w] < 0) {
				a->back[w] = a->back[u] + 1;
				a->queue[tail++] = w;
			}
		}
	}
	*np = 0;
	*stop = 0;
	if (a->back[s] < 0) {
		return ORC_OK; /* NULL */
	}
	drop_layers(a);
	int64_t *w0 = new_layer(a);
	if (!w0) {
		return ORC_ERR_ALLOC;
	}
	w0[s] = 1;
	/* the count of each layer at t, and the layers' walks once the last one is known */
	int64_t total = s == t ? 1 : 0;
	int64_t H = 0;
	while (total < kk) {
		const int64_t h = a->nlayers;
		const int64_t *prev = a->layer[h - 1];
		int64_t *cur = new_layer(a);
		if (!cur) {
			return ORC_ERR_ALLOC;
		}
		int alive = 0;
		for (int64_t q = 0; q < tail; q++) { /* the vertices of B(t) */
			const int64_t u = a->queue[q];
			int64_t sum = 0;
			for (int64_t j = a->in_off[u]; j < a->in_off[u + 1]; j++) {
				sum = sat_add(sum, prev[a->in_src[j]]);
			}
			cur[u] = sum;
			alive |= sum != 0;
		}
		*stop = h;
		if (cur[t] > 0) {
			if (h > ORC_WALK_MAX) {
				return ORC_ERR_UNSUPPORTED;
			}
			total = sat_add(total, cur[t]);
			H = h;
		}
		if (!alive) {
			break;
		}
		if (total < kk && h > ORC_WALK_MAX) {
			return ORC_ERR_UNSUPPORTED; /* a longer walk to t exists and is needed */
		}
	}
	/* the walks, length by length */
	int64_t left = kk;
	for (int64_t h = 0; h <= H && left > 0; h++) {
		const int64_t c = a->layer[h][t];
		const int64_t want = c < left ? c : left;
		if (want > 0) {
			int rc = enumerate(a, t, h, want);
			if (rc) {
				return rc;
			}
			left -= want;
			*np += want;
		}
	}
	return ORC_OK;
}

/* Row i: out_valid, out_npaths walks from walk out_first[i] on; walk j is (*out_elems)[(*out_offsets)[j] ..
 * (*out_offsets)[j + 1]).  stats (6 entries): batches, lanes, searches, levels, push_levels, walks. */
int orc_shortest_k_paths(int64_t n, const int64_t *v, const int64_t *e, const int64_t *edge_ids, int64_t p,
                         const int64_t *src, const int64_t *dst, const uint8_t *src_valid, const uint8_t *dst_valid,
                         int64_t k, int64_t lanes, int64_t *out_npaths, int64_t *out_first, uint8_t *out_valid,
                         int64_t **out_offsets, int64_t **out_elems, int64_t *stats) {
	if (n < 0 || p < 0 || k < 1 || lanes < 1) {
		return ORC_ERR_ARG;
	}
	int rc = ORC_OK;
	const int64_t m = v[n];
	orc_ks a;
	memset(&a, 0, sizeof(a));
	a.n = n;
	a.edge_ids = edge_ids;
	vec elems = {0, 0, 0}, offsets = {0, 0, 0};
	a.elems = &elems;
	a.offsets = &offsets;
	a.in_off = (int64_t *)calloc((size_t)n + 2, sizeof(int64_t));
	a.in_src = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.in_idx = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.back = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.queue = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.path = (int64_t *)malloc((2 * (size_t)ORC_WALK_MAX + 4) * sizeof(int64_t));
	a.cursor = (int64_t *)malloc(((size_t)ORC_WALK_MAX + 3) * sizeof(int64_t));
	int64_t *fill = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
	if (!a.in_off || !a.in_src || !a.in_idx || !a.back || !a.queue || !a.path || !a.cursor || !fill) {
		rc = ORC_ERR_ALLOC;
		goto done;
	}
	for (int64_t idx = 0; idx < m; idx++) {
		a.in_off[e[idx] + 1]++;
	}
	for (int64_t u = 0; u < n; u++) {
		a.in_off[u + 1] += a.in_off[u];
	}
	for (int64_t row = 0; row < n; row++) {
		for (int64_t idx = v[row]; idx < v[row + 1]; idx++) {
			const int64_t x = a.in_off[e[idx]] + fill[e[idx]]++;
			a.in_src[x] = row;
			a.in_idx[x] = idx;
		}
	}
	for (int64_t i = 0; i < p; i++) {
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		if (src[i] < 0 || src[i] >= n || dst[i] < 0 || dst[i] >= n) {
			rc = ORC_ERR_RANGE;
			goto done;
		}
	}
	memset(stats, 0, 6 * sizeof(int64_t));
	stats[1] = lanes;
	int64_t lane = 0, batch_levels = 0, batch_push = 0;
	for (int64_t i = 0; i < p; i++) {
		out_npaths[i] = 0;
		out_first[i] = offsets.size;
		out_valid[i] = 0;
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		int64_t np, stop, ecc;
		rc = one_row(&a, src[i], dst[i], k, &np, &stop, &ecc);
		if (rc) {
			goto done;
		}
		out_npaths[i] = np;
		out_valid[i] = np > 0;
		batch_levels = stop > batch_levels ? stop : batch_levels;
		batch_push = ecc + 1 > batch_push ? ecc + 1 : batch_push;
		stats[2]++;
		if (++lane == lanes) { /* a full batch */
			lane = 0;
			stats[0]++;
			stats[3] += batch_levels;
			stats[4] += batch_push;
			batch_levels = batch_push = 0;
		}
	}
	if (lane > 0) {
		stats[0]++;
		stats[3] += batch_levels;
		stats[4] += batch_push;
	}
	stats[5] = offsets.size;
	if (vec_push(&offsets, elems.size)) {
		rc = ORC_ERR_ALLOC;
		goto done;
	}
	*out_offsets = offsets.data;
	*out_elems = elems.data;
	offsets.data = NULL;
	elems.data = NULL;
done:
	drop_layers(&a);
	free(a.layer);
	free(offsets.data);
	free(elems.data);
	free(a.in_off);
	free(a.in_src);
	free(a.in_idx);
	free(a.back);
	free(a.queue);
	free(a.path);
	free(a.cursor);
	free(fill);
	return rc;
}

void orc_kshortest_free(void *x) {
	free(x);
}
