/*
 * pgq_oracle_allshortest.c -- CPU restatement of shortest_path_count and all_shortest_paths, AN EXTENSION: the
 * reference has no such function (it rejects ALL SHORTEST).
 *
 * TEST INFRASTRUCTURE ONLY, like pgq_oracle.c: the checker of pgq_shortest_path_count and pgq_all_shortest_paths.
 * Only tests/ and tools/ may build, load or call this file; the product never links or falls back to it.
 *
 * Written from the definitions in include/duckpgq_b200.h alone, over the reference CSR layout (v offsets, e targets,
 * edge ids, original vertex ids):
 *   - one sequential BFS per distinct source gives dist; sigma(s) = 1 and, visiting the vertices in BFS order, every
 *     out-edge u -> w with dist(w) = dist(u) + 1 adds sigma(u) to sigma(w), saturating at INT64_MAX;
 *   - count(s, t) = sigma(t) (1 for s == t), NULL when t is not reached or an id is NULL;
 *   - the paths are enumerated by a depth-first search back from t that tries, at a node of depth k, its in-edges from
 *     vertices of depth k - 1 in step order (the parent's id, then the edge's position in the parent's adjacency) and
 *     stops after max_paths complete paths (0 = all of them).  The device unranks instead; the two meet only in the
 *     order both are defined by.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_ERR_ALLOC 1
#define ORC_ERR_ARG 2
#define ORC_ERR_RANGE 3
#define ORC_ERR_UNSUPPORTED 4

#define ORC_DEPTH_MAX 65533 /* the device's path mode records levels up to this depth */

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

/* the in-lists in step order: in_src[k], in_idx[k] for k in [in_off[u], in_off[u + 1]), sorted by (source row,
 * position), which is the order a sweep over the rows and their adjacencies produces */
typedef struct {
	int64_t n;
	const int64_t *v, *e, *edge_ids;
	int64_t *in_off, *in_src, *in_idx;
	int64_t *dist, *sigma, *queue;
	/* the walk of the enumeration */
	int64_t *path;   /* [2 h + 1] */
	int64_t *cursor; /* [h + 1] */
	int64_t limit, emitted;
	vec *out;
} orc_as;

/* the paths back from t at depth h, depth first: cursor[k] is the next in-list entry to try at the node of depth k
 * (path[2k]); stops after a->limit complete paths when a->limit > 0 */
static int enumerate(orc_as *a, int64_t t, int64_t h, int64_t len) {
	int64_t k = h;
	a->path[2 * h] = t;
	a->cursor[h] = a->in_off[t];
	while (k <= h) {
		if (k == 0) {
			for (int64_t i = 0; i < len; i++) {
				if (vec_push(a->out, a->path[i])) {
					return ORC_ERR_ALLOC;
				}
			}
			if (++a->emitted == a->limit) {
				return ORC_OK;
			}
			k = 1;
			continue;
		}
		const int64_t u = a->path[2 * k];
		int64_t j = a->cursor[k];
		while (j < a->in_off[u + 1] && a->dist[a->in_src[j]] != k - 1) {
			j++;
		}
		if (j == a->in_off[u + 1]) {
			k++; /* every parent of this node tried: back one step */
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

static void bfs(orc_as *a, int64_t s) {
	const int64_t n = a->n;
	for (int64_t i = 0; i < n; i++) {
		a->dist[i] = -1;
		a->sigma[i] = 0;
	}
	int64_t head = 0, tail = 0;
	a->dist[s] = 0;
	a->sigma[s] = 1;
	a->queue[tail++] = s;
	while (head < tail) {
		const int64_t u = a->queue[head++];
		for (int64_t idx = a->v[u]; idx < a->v[u + 1]; idx++) {
			const int64_t w = a->e[idx];
			if (a->dist[w] < 0) {
				a->dist[w] = a->dist[u] + 1;
				a->queue[tail++] = w;
			}
			if (a->dist[w] == a->dist[u] + 1) {
				a->sigma[w] = sat_add(a->sigma[w], a->sigma[u]);
			}
		}
	}
}

static const int64_t *g_src; /* (qsort's comparison of rows by source) */
static int by_source(const void *x, const void *y) {
	const int64_t a = g_src[*(const int64_t *)x], b = g_src[*(const int64_t *)y];
	if (a != b) {
		return a < b ? -1 : 1;
	}
	return *(const int64_t *)x < *(const int64_t *)y ? -1 : 1;
}

/* lists = 0: counts only (out_npaths, out_path_len, out_offsets, out_elems, out_total unused).
 * Row i: out_count, out_valid; with lists, out_npaths[i] paths of out_path_len[i] elements from (*out_elems)[out_offsets[i]]. */
int orc_all_shortest_paths(int64_t n, const int64_t *v, const int64_t *e, const int64_t *edge_ids, int64_t p,
                           const int64_t *src, const int64_t *dst, const uint8_t *src_valid, const uint8_t *dst_valid,
                           int64_t max_paths, int lists, int64_t *out_count, int64_t *out_npaths, int64_t *out_path_len,
                           int64_t *out_offsets, uint8_t *out_valid, int64_t **out_elems, int64_t *out_total) {
	if (n < 0 || p < 0 || max_paths < 0) {
		return ORC_ERR_ARG;
	}
	int rc = ORC_OK;
	const int64_t m = v[n];
	orc_as a;
	memset(&a, 0, sizeof(a));
	a.n = n;
	a.v = v;
	a.e = e;
	a.edge_ids = edge_ids;
	vec out = {0, 0, 0};
	a.out = &out;
	a.in_off = (int64_t *)calloc((size_t)n + 2, sizeof(int64_t));
	a.in_src = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.in_idx = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.dist = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.sigma = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.queue = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.path = (int64_t *)malloc((2 * (size_t)ORC_DEPTH_MAX + 2) * sizeof(int64_t));
	a.cursor = (int64_t *)malloc(((size_t)ORC_DEPTH_MAX + 2) * sizeof(int64_t));
	int64_t *order = (int64_t *)malloc(((size_t)p + 1) * sizeof(int64_t));
	int64_t *fill = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
	if (!a.in_off || !a.in_src || !a.in_idx || !a.dist || !a.sigma || !a.queue || !a.path || !a.cursor || !order || !fill) {
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
			const int64_t k = a.in_off[e[idx]] + fill[e[idx]]++;
			a.in_src[k] = row;
			a.in_idx[k] = idx;
		}
	}
	/* the rows that search, grouped by source (one BFS per distinct source) */
	int64_t searching = 0;
	for (int64_t i = 0; i < p; i++) {
		out_count[i] = 0;
		out_valid[i] = 0;
		if (lists) {
			out_npaths[i] = 0;
			out_path_len[i] = 0;
		}
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		if (src[i] < 0 || src[i] >= n || dst[i] < 0 || dst[i] >= n) {
			rc = ORC_ERR_RANGE;
			goto done;
		}
		order[searching++] = i;
	}
	g_src = src;
	qsort(order, (size_t)searching, sizeof(int64_t), by_source);
	for (int64_t k = 0; k < searching; k++) {
		const int64_t i = order[k];
		if (k == 0 || src[order[k - 1]] != src[i]) {
			bfs(&a, src[i]);
		}
		const int64_t t = dst[i], h = a.dist[t];
		if (h < 0) {
			continue;
		}
		if (h > ORC_DEPTH_MAX) {
			rc = ORC_ERR_UNSUPPORTED;
			goto done;
		}
		out_count[i] = a.sigma[t];
		out_valid[i] = 1;
	}
	if (lists) {
		/* enumerate in row order, each row by the BFS of its source again (rows of one source in a row share it) */
		int64_t last = -1;
		for (int64_t i = 0; i < p; i++) {
			if (!out_valid[i]) {
				continue;
			}
			if (max_paths == 0 && out_count[i] == INT64_MAX) {
				rc = ORC_ERR_UNSUPPORTED;
				goto done;
			}
			if (src[i] != last) {
				bfs(&a, src[i]);
				last = src[i];
			}
			const int64_t h = a.dist[dst[i]], len = 2 * h + 1;
			a.limit = max_paths;
			a.emitted = 0;
			rc = enumerate(&a, dst[i], h, len);
			if (rc) {
				goto done;
			}
			out_npaths[i] = a.emitted;
			out_path_len[i] = len;
		}
		int64_t pos = 0;
		for (int64_t i = 0; i < p; i++) {
			out_offsets[i] = pos;
			pos += out_npaths[i] * out_path_len[i];
		}
		*out_elems = out.data;
		*out_total = out.size;
		out.data = NULL;
	}
done:
	free(out.data);
	free(a.in_off);
	free(a.in_src);
	free(a.in_idx);
	free(a.dist);
	free(a.sigma);
	free(a.queue);
	free(a.path);
	free(a.cursor);
	free(order);
	free(fill);
	return rc;
}

void orc_allshortest_free(void *x) {
	free(x);
}
