/*
 * pgq_oracle_allcheapest.c -- CPU restatement of cheapest_path_count and all_cheapest_paths, AN EXTENSION: the
 * reference has no such functions (SQL/PGQ's ALL CHEAPEST).
 *
 * TEST INFRASTRUCTURE ONLY, like pgq_oracle.c: the checker of pgq_cheapest_path_count / pgq_all_cheapest_paths.  Only
 * tests/ and tools/ may build, load or call this file; the product never links or falls back to it.
 *
 * Rows take lanes in input order, `lanes` per batch.  Each batch runs the Bellman-Ford sweeps of cheapest_path_length
 * (ORC_BF_SWEEPS of pgq_oracle_cheapest.c, included below) to the distances d, which decide for each lane which edges
 * are tight (d(v) + w == d(u) in the weight type's arithmetic: orc_tight_i64 / orc_tight_f64).  Then, one lane at a time:
 *   - open: both ids valid, and s == t or d(t) is not the sentinel max/2;
 *   - B(t): a breadth-first search back from t over the lane's tight in-edges; s outside B(t) makes the row NULL;
 *   - counts: w_0 = [s], w_h(u) = the sum of w_{h-1}(v) over the tight in-edges v -> u, kept for u in B(t) only,
 *     saturating at INT64_MAX.  After layer h the lane adds w_h(t) to its total and lists min(w_h(t), the room under
 *     max_paths) paths of h edges (all for max_paths = 0, none for a count); it stops when w_h is zero on B(t), when its
 *     total saturates, or once w_h is non-zero at h >= |B(t)| (infinitely many: count INT64_MAX) -- then at once for a
 *     count or max_paths = 0, else when it has max_paths paths;
 *   - the lists: for each length h, a depth-first search back from t over the step lists (in-edges sorted by the
 *     parent's id, then the edge's position in the parent's adjacency), entering only tight edges whose parent has
 *     w_{j-1} > 0 with j steps left, so that the paths come out in the order of the header and every branch ends in one.
 * stats: batches; push_levels = the sum over batches of 1 + the largest tight distance to an open lane's target;
 * pull_levels = the sum over batches of the largest stopping layer of a lane that counted; walks = paths listed.
 */
#include "pgq_oracle_cheapest.c"

#define AC_MAX INT64_MAX
#define AC_WALK_MAX 65533

typedef struct {
	int64_t batches;
	int64_t push_levels;
	int64_t pull_levels;
	int64_t walks;
} orc_ac_stats;

static inline uint64_t ac_sat(uint64_t a, uint64_t b) {
	return a > (uint64_t)AC_MAX - b ? (uint64_t)AC_MAX : a + b;
}

typedef struct { /* a growing int64 array */
	int64_t *a;
	size_t n, cap;
} ac_vec;

static int ac_push(ac_vec *v, int64_t x) {
	if (v->n == v->cap) {
		size_t cap = v->cap ? 2 * v->cap : 1024;
		int64_t *a = (int64_t *)realloc(v->a, cap * sizeof(int64_t));
		if (!a) {
			return ORC_ERR_ALLOC;
		}
		v->a = a;
		v->cap = cap;
	}
	v->a[v->n++] = x;
	return ORC_OK;
}

/* What the generic part reads: the graph, its step lists, and the batch's tight table tight[l * m + index] */
typedef struct {
	int64_t n, m;
	const int64_t *v, *e, *edge_ids;
	const int64_t *in_off, *in_par, *in_idx; /* step lists: u's in-edges at [in_off[u], in_off[u + 1]) */
	const uint8_t *tight;
	int64_t walks_limit;
} ac_graph;

/* Depth-first listing of the paths of h edges from s to t, at most `want` of them, into elems / offs */
typedef struct {
	const ac_graph *g;
	int lane;
	int64_t s;
	uint64_t **layers; /* layers[j - 1] = w_j over all vertices */
	int64_t *stack_v, *stack_e;
	int64_t want, got;
	ac_vec *elems, *offs;
	int rc;
} ac_dfs;

static void ac_dfs_go(ac_dfs *d, int64_t u, int j, int h) {
	if (d->got >= d->want || d->rc) {
		return;
	}
	if (j == 0) { /* u == s: emit [s, e1, v1, ..., eh, t] */
		if (ac_push(d->offs, (int64_t)d->elems->n)) {
			d->rc = ORC_ERR_ALLOC;
			return;
		}
		int rc = ac_push(d->elems, d->s);
		for (int k = 1; k <= h && !rc; k++) {
			rc = ac_push(d->elems, d->stack_e[k]);
			if (!rc) {
				rc = ac_push(d->elems, d->stack_v[k]);
			}
		}
		d->rc = rc;
		d->got++;
		return;
	}
	const ac_graph *g = d->g;
	for (int64_t x = g->in_off[u]; x < g->in_off[u + 1] && d->got < d->want && !d->rc; x++) {
		const int64_t par = g->in_par[x], idx = g->in_idx[x];
		if (!g->tight[(size_t)d->lane * (size_t)g->m + (size_t)idx]) {
			continue;
		}
		const uint64_t wv = j == 1 ? (par == d->s) : d->layers[j - 2][par];
		if (!wv) {
			continue;
		}
		d->stack_v[j] = u;
		d->stack_e[j] = g->edge_ids[idx];
		ac_dfs_go(d, par, j - 1, h);
	}
}

/* One lane: reach, counts, lists.  Returns its stopping layer in *stop_h (0: it did not count), its reach depth in
 * *depth (-1: not open). */
static int ac_lane(const ac_graph *g, int lane, int open, int64_t s, int64_t t, int list, int64_t max_paths,
                   int64_t *out_count, int64_t *out_npaths, ac_vec *elems, ac_vec *offs, int64_t *stop_h,
                   int64_t *depth) {
	const int64_t n = g->n;
	*out_count = 0;
	*out_npaths = 0;
	*stop_h = 0;
	*depth = -1;
	if (!open) {
		return ORC_OK;
	}
	int rc = ORC_OK;
	int32_t *dist = (int32_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(int32_t));
	int64_t *queue = (int64_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(int64_t));
	uint64_t *prev = (uint64_t *)calloc((size_t)(n > 0 ? n : 1), sizeof(uint64_t));
	uint64_t *cur = (uint64_t *)calloc((size_t)(n > 0 ? n : 1), sizeof(uint64_t));
	uint64_t **layers = NULL;
	int64_t *takes = NULL, nlayers = 0, cap_layers = 0;
	if (!dist || !queue || !prev || !cur) {
		rc = ORC_ERR_ALLOC;
		goto out;
	}
	/* B(t): back from t over the tight in-edges */
	for (int64_t i = 0; i < n; i++) {
		dist[i] = -1;
	}
	int64_t qh = 0, qt = 0, bsize = 0, maxd = 0;
	dist[t] = 0;
	queue[qt++] = t;
	while (qh < qt) {
		const int64_t u = queue[qh++];
		bsize++;
		if (dist[u] > maxd) {
			maxd = dist[u];
		}
		for (int64_t x = g->in_off[u]; x < g->in_off[u + 1]; x++) {
			const int64_t par = g->in_par[x];
			if (g->tight[(size_t)lane * (size_t)g->m + (size_t)g->in_idx[x]] && dist[par] < 0) {
				dist[par] = dist[u] + 1;
				queue[qt++] = par;
			}
		}
	}
	*depth = maxd;
	if (dist[s] < 0) {
		goto out; /* NULL */
	}
	/* the counting layers; queue[0 .. bsize) lists B(t) */
	uint64_t total = s == t ? 1 : 0;
	int64_t listed = list && s == t ? 1 : 0;
	int inf = 0;
	for (int64_t h = 1;; h++) {
		int alive = 0;
		for (int64_t q = 0; q < bsize; q++) {
			const int64_t u = queue[q];
			uint64_t sum = 0;
			for (int64_t x = g->in_off[u]; x < g->in_off[u + 1]; x++) {
				const int64_t par = g->in_par[x];
				if (g->tight[(size_t)lane * (size_t)g->m + (size_t)g->in_idx[x]]) {
					sum = ac_sat(sum, h == 1 ? (uint64_t)(par == s) : prev[par]);
				}
			}
			cur[u] = sum;
			alive |= sum != 0;
		}
		const uint64_t c = cur[t];
		total = ac_sat(total, c);
		uint64_t take = 0;
		if (list) {
			take = max_paths ? (c < (uint64_t)(max_paths - listed) ? c : (uint64_t)(max_paths - listed)) : c;
			listed = (int64_t)ac_sat((uint64_t)listed, take);
		}
		if (list) { /* keep the layer for the listing */
			if (nlayers == cap_layers) {
				cap_layers = cap_layers ? 2 * cap_layers : 16;
				uint64_t **l2 = (uint64_t **)realloc(layers, (size_t)cap_layers * sizeof(uint64_t *));
				int64_t *t2 = (int64_t *)realloc(takes, (size_t)cap_layers * sizeof(int64_t));
				if (l2) {
					layers = l2;
				}
				if (t2) {
					takes = t2;
				}
				if (!l2 || !t2) {
					rc = ORC_ERR_ALLOC;
					goto out;
				}
			}
			layers[nlayers] = (uint64_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(uint64_t));
			if (!layers[nlayers]) {
				rc = ORC_ERR_ALLOC;
				goto out;
			}
			memcpy(layers[nlayers], cur, (size_t)n * sizeof(uint64_t));
			takes[nlayers] = (int64_t)take;
			nlayers++;
		}
		inf = inf || (alive && (uint64_t)h >= (uint64_t)bsize);
		const int stop = !alive || total == (uint64_t)AC_MAX ||
		                 (inf && (!list || max_paths == 0 || listed >= max_paths));
		if (h >= AC_WALK_MAX && !stop) {
			rc = ORC_ERR_UNSUPPORTED;
			goto out;
		}
		*stop_h = h;
		if (stop) {
			break;
		}
		uint64_t *tmp = prev;
		prev = cur;
		cur = tmp;
		for (int64_t q = 0; q < bsize; q++) {
			cur[queue[q]] = 0;
		}
	}
	*out_count = inf ? AC_MAX : (int64_t)total;
	if (!list) {
		goto out;
	}
	if (max_paths == 0 && *out_count == AC_MAX) {
		rc = ORC_ERR_UNSUPPORTED;
		goto out;
	}
	*out_npaths = listed;
	if (s == t) { /* [s] */
		if (ac_push(offs, (int64_t)elems->n) || ac_push(elems, s)) {
			rc = ORC_ERR_ALLOC;
			goto out;
		}
	}
	{
		int64_t *sv = (int64_t *)malloc((size_t)(nlayers + 2) * sizeof(int64_t));
		int64_t *se = (int64_t *)malloc((size_t)(nlayers + 2) * sizeof(int64_t));
		if (!sv || !se) {
			free(sv);
			free(se);
			rc = ORC_ERR_ALLOC;
			goto out;
		}
		for (int64_t h = 1; h <= nlayers && !rc; h++) {
			if (!takes[h - 1]) {
				continue;
			}
			ac_dfs d = {g, lane, s, layers, sv, se, takes[h - 1], 0, elems, offs, ORC_OK};
			ac_dfs_go(&d, t, (int)h, (int)h);
			rc = d.rc;
		}
		free(sv);
		free(se);
	}
out:
	for (int64_t i = 0; i < nlayers; i++) {
		free(layers[i]);
	}
	free(layers);
	free(takes);
	free(dist);
	free(queue);
	free(prev);
	free(cur);
	return rc;
}

/* The sweeps and the tight table of one batch (typed), then the lanes (generic) */
#define ORC_ALL_CHEAPEST_BODY(T, INF, TIGHT)                                                                       \
	if (lanes <= 0 || max_paths < 0) {                                                                             \
		return ORC_ERR_ARG;                                                                                        \
	}                                                                                                              \
	orc_ac_stats local;                                                                                            \
	memset(&local, 0, sizeof(local));                                                                              \
	const int lane_limit = lanes;                                                                                  \
	const int64_t m = v[v_size];                                                                                   \
	const size_t cells = (size_t)(v_size > 0 ? v_size : 1) * lanes;                                                \
	T *dists = (T *)malloc(cells * sizeof(T));                                                                     \
	uint8_t *tight = (uint8_t *)malloc((size_t)lanes * (size_t)(m > 0 ? m : 1));                                   \
	uint8_t *open = (uint8_t *)malloc((size_t)lanes);                                                              \
	int64_t *in_off = (int64_t *)calloc((size_t)v_size + 2, sizeof(int64_t));                                      \
	int64_t *in_par = (int64_t *)malloc((size_t)(m > 0 ? m : 1) * sizeof(int64_t));                                \
	int64_t *in_idx = (int64_t *)malloc((size_t)(m > 0 ? m : 1) * sizeof(int64_t));                                \
	ac_vec elems = {NULL, 0, 0}, offs = {NULL, 0, 0};                                                              \
	int rc = ORC_OK;                                                                                               \
	if (!dists || !tight || !open || !in_off || !in_par || !in_idx) {                                              \
		rc = ORC_ERR_ALLOC;                                                                                        \
		goto done;                                                                                                 \
	}                                                                                                              \
	/* the step lists: parents ascending, then their adjacency positions ascending */                              \
	for (int64_t index = 0; index < m; index++) {                                                                  \
		in_off[e[index] + 1]++;                                                                                    \
	}                                                                                                              \
	for (int64_t u = 0; u < v_size; u++) {                                                                         \
		in_off[u + 1] += in_off[u];                                                                                \
	}                                                                                                              \
	{                                                                                                              \
		int64_t *fill = (int64_t *)malloc((size_t)(v_size > 0 ? v_size : 1) * sizeof(int64_t));                   \
		if (!fill) {                                                                                               \
			rc = ORC_ERR_ALLOC;                                                                                    \
			goto done;                                                                                             \
		}                                                                                                          \
		memcpy(fill, in_off, (size_t)v_size * sizeof(int64_t));                                                    \
		for (int64_t vv = 0; vv < v_size; vv++) {                                                                  \
			for (int64_t index = v[vv]; index < v[vv + 1]; index++) {                                             \
				in_par[fill[e[index]]] = vv;                                                                       \
				in_idx[fill[e[index]]++] = index;                                                                  \
			}                                                                                                      \
		}                                                                                                          \
		free(fill);                                                                                                \
	}                                                                                                              \
	const ac_graph g = {v_size, m, v, e, edge_ids, in_off, in_par, in_idx, tight, 0};                              \
	for (int64_t b0 = 0; b0 < p; b0 += lanes) {                                                                    \
		const int cnt = (int)(p - b0 < lanes ? p - b0 : lanes);                                                    \
		for (size_t i = 0; i < cells; i++) {                                                                       \
			dists[i] = (INF);                                                                                      \
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
		for (int l = 0; l < cnt; l++) {                                                                            \
			for (int64_t vv = 0; vv < v_size; vv++) {                                                              \
				for (int64_t index = v[vv]; index < v[vv + 1]; index++) {                                          \
					tight[(size_t)l * (size_t)m + (size_t)index] =                                                 \
					    (uint8_t)TIGHT(dists[vv * lanes + l], w[index], dists[e[index] * lanes + l]);              \
				}                                                                                                  \
			}                                                                                                      \
			int64_t row = b0 + l;                                                                                  \
			open[l] = (!src_valid || src_valid[row]) && (!dst_valid || dst_valid[row]) &&                          \
			          (src[row] == dst[row] || dists[dst[row] * lanes + l] != (INF));                              \
		}                                                                                                          \
		int64_t push = 0, pull = 0;                                                                                \
		for (int l = 0; l < cnt && !rc; l++) {                                                                     \
			int64_t row = b0 + l, stop_h = 0, depth = -1;                                                          \
			out_first[row] = (int64_t)offs.n;                                                                      \
			rc = ac_lane(&g, l, open[l], open[l] ? src[row] : 0, open[l] ? dst[row] : 0, list, max_paths,          \
			             &out_count[row], &out_npaths[row], &elems, &offs, &stop_h, &depth);                       \
			out_valid[row] = out_count[row] > 0;                                                                   \
			push = depth > push ? depth : push;                                                                    \
			pull = stop_h > pull ? stop_h : pull;                                                                  \
		}                                                                                                          \
		if (rc) {                                                                                                  \
			goto done;                                                                                             \
		}                                                                                                          \
		local.push_levels += push + 1;                                                                             \
		local.pull_levels += pull;                                                                                 \
	}                                                                                                              \
	local.walks = (int64_t)offs.n;                                                                                 \
	if (ac_push(&offs, (int64_t)elems.n) || (!elems.a && ac_push(&elems, 0))) {                                    \
		rc = ORC_ERR_ALLOC;                                                                                        \
	}                                                                                                              \
done:                                                                                                              \
	if (stats) {                                                                                                   \
		*stats = local;                                                                                            \
	}                                                                                                              \
	free(dists);                                                                                                   \
	free(tight);                                                                                                   \
	free(open);                                                                                                    \
	free(in_off);                                                                                                  \
	free(in_par);                                                                                                  \
	free(in_idx);                                                                                                  \
	if (rc != ORC_OK) {                                                                                            \
		free(elems.a);                                                                                             \
		free(offs.a);                                                                                              \
		elems.a = offs.a = NULL;                                                                                   \
	}                                                                                                              \
	*out_elems = elems.a;                                                                                          \
	*out_offsets = offs.a;                                                                                         \
	return rc;

int orc_all_cheapest_paths_i64(int64_t v_size, const int64_t *v, const int64_t *e, const int64_t *edge_ids,
                               const int64_t *w, int64_t p, const int64_t *src, const int64_t *dst,
                               const uint8_t *src_valid, const uint8_t *dst_valid, int lanes, int list,
                               int64_t max_paths, int64_t *out_count, int64_t *out_npaths, int64_t *out_first,
                               uint8_t *out_valid, int64_t **out_offsets, int64_t **out_elems, orc_ac_stats *stats) {
	ORC_ALL_CHEAPEST_BODY(int64_t, INT64_MAX / 2, orc_tight_i64)
}

int orc_all_cheapest_paths_f64(int64_t v_size, const int64_t *v, const int64_t *e, const int64_t *edge_ids,
                               const double *w, int64_t p, const int64_t *src, const int64_t *dst,
                               const uint8_t *src_valid, const uint8_t *dst_valid, int lanes, int list,
                               int64_t max_paths, int64_t *out_count, int64_t *out_npaths, int64_t *out_first,
                               uint8_t *out_valid, int64_t **out_offsets, int64_t **out_elems, orc_ac_stats *stats) {
	ORC_ALL_CHEAPEST_BODY(double, 1.7976931348623157e308 / 2, orc_tight_f64)
}
