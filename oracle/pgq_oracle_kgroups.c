/*
 * pgq_oracle_kgroups.c -- CPU restatement of shortest_k_groups, AN EXTENSION: the reference carries SQL/PGQ's
 * SHORTEST k GROUP in its AST (PathPattern::group) and rejects it before acting on it.
 *
 * TEST INFRASTRUCTURE ONLY, like pgq_oracle.c: the checker of pgq_shortest_k_groups.  Only tests/ and tools/ may build,
 * load or call this file; the product never links or falls back to it.
 *
 * Written from the definitions in include/duckpgq_b200.h alone, over the reference CSR layout (v offsets, e targets,
 * edge ids, original vertex ids), one row at a time:
 *   - WALK: B(t) by a sequential BFS back from t; the layers w_h(u) = the number of h-edge walks s -> u on B(t),
 *     saturated at INT64_MAX, every layer kept; a row stops after its k-th length group or after a layer that is zero
 *     on all of B(t).  The walks of each group length are enumerated by a depth-first search back from t in step
 *     order, until max_paths are listed.  The stats simulate the batches at the lane width.
 *   - TRAIL, ACYCLIC, SIMPLE: Yen's algorithm with Lawler's rule, a plain BFS per spur search and a sorted array as the
 *     pool; before it accepts its pool's least path a row stops when the pool is empty, when it has k groups and the
 *     least path is longer than its last group's length, or when it lists max_paths paths already (then complete
 *     exactly when the least path is not part of the result).  The stats simulate the rounds and their batches.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_ERR_ALLOC 1
#define ORC_ERR_ARG 2
#define ORC_ERR_RANGE 3
#define ORC_ERR_UNSUPPORTED 4

#define ORC_PATH_MAX 65533 /* the longest path a result may hold */
#define ORC_WALK 0
#define ORC_TRAIL 1
#define ORC_ACYCLIC 2
#define ORC_SIMPLE 3
#define ORC_BUDGET ((int64_t)4 << 30)

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

/* a path: h edges; vert[0..h] original vertex ids, pos[0..h) CSR positions, dev its spur index */
typedef struct {
	int64_t h, dev;
	int64_t *vert, *pos;
} path;

static void path_free(path *p) {
	free(p->vert);
	free(p->pos);
	p->vert = p->pos = NULL;
}

/* the result's order: h, then (parent, position) from t back to s */
static int path_cmp(const path *a, const path *b) {
	if (a->h != b->h) {
		return a->h < b->h ? -1 : 1;
	}
	for (int64_t i = a->h - 1; i >= 0; i--) {
		if (a->vert[i] != b->vert[i]) {
			return a->vert[i] < b->vert[i] ? -1 : 1;
		}
		if (a->pos[i] != b->pos[i]) {
			return a->pos[i] < b->pos[i] ? -1 : 1;
		}
	}
	return 0;
}

typedef struct {
	int64_t n, m;
	const int64_t *v, *e, *edge_ids;
	int64_t *in_off, *in_src, *in_idx; /* in-lists in step order */
	vec *elems, *offsets;
	/* WALK */
	int64_t *back, *bq;  /* BFS back from t: depth (-1: does not reach t) and its queue */
	int64_t **layer;     /* layer[h][u] = w_h(u) */
	int64_t nlayers, cap_layers;
	int64_t *wpath, *cursor;
	/* the modes */
	int64_t *lvl, *queue, *nextq;
	int64_t *vban, *eban, *dban; /* stamps */
	int64_t stamp;
	int64_t *sp_pos, *sp_vert;
	path *acc, *pool;
	int64_t nacc, npool, cap_acc, cap_pool;
	vec *round_x; /* per round: the expansions of each search that took a lane */
	int64_t nrounds;
} orc_kg;

/* one row's results */
typedef struct {
	int64_t count, ngroups, last, npaths;
	int complete;
} kg_row;

/* ---- WALK ---- */

static int64_t *new_layer(orc_kg *a) {
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

static void drop_layers(orc_kg *a) {
	for (int64_t i = 0; i < a->nlayers; i++) {
		free(a->layer[i]);
	}
	a->nlayers = 0;
}

/* the first `want` walks of h edges s -> t in step order */
static int enumerate(orc_kg *a, int64_t t, int64_t h, int64_t want) {
	const int64_t len = 2 * h + 1;
	int64_t got = 0, k = h;
	a->wpath[2 * h] = t;
	a->cursor[h] = a->in_off[t];
	while (k <= h && got < want) {
		if (k == 0) {
			if (vec_push(a->offsets, a->elems->size)) {
				return ORC_ERR_ALLOC;
			}
			for (int64_t i = 0; i < len; i++) {
				if (vec_push(a->elems, a->wpath[i])) {
					return ORC_ERR_ALLOC;
				}
			}
			got++;
			k = 1;
			continue;
		}
		const int64_t u = a->wpath[2 * k];
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
		a->wpath[2 * k - 1] = a->edge_ids[a->in_idx[j]];
		a->wpath[2 * k - 2] = par;
		k--;
		a->cursor[k] = a->in_off[par];
	}
	return ORC_OK;
}

/* one WALK row: *stop = the last layer computed (0 when none was), *ecc = the depth of the BFS back from t */
static int walk_row(orc_kg *a, int64_t s, int64_t t, int64_t k, int64_t max_paths, int count_only, kg_row *r,
                    int64_t *stop, int64_t *ecc) {
	const int64_t n = a->n;
	for (int64_t u = 0; u < n; u++) {
		a->back[u] = -1;
	}
	int64_t head = 0, tail = 0;
	a->back[t] = 0;
	a->bq[tail++] = t;
	*ecc = 0;
	while (head < tail) {
		const int64_t u = a->bq[head++];
		*ecc = a->back[u];
		for (int64_t j = a->in_off[u]; j < a->in_off[u + 1]; j++) {
			const int64_t w = a->in_src[j];
			if (a->back[w] < 0) {
				a->back[w] = a->back[u] + 1;
				a->bq[tail++] = w;
			}
		}
	}
	memset(r, 0, sizeof(*r));
	r->last = -1;
	r->complete = 1;
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
	if (s == t) {
		r->count = r->ngroups = 1;
		r->last = 0;
	}
	while (r->ngroups < k) {
		const int64_t h = a->nlayers;
		const int64_t *prev = a->layer[h - 1];
		int64_t *cur = new_layer(a);
		if (!cur) {
			return ORC_ERR_ALLOC;
		}
		int alive = 0;
		for (int64_t q = 0; q < tail; q++) { /* the vertices of B(t) */
			const int64_t u = a->bq[q];
			int64_t sum = 0;
			for (int64_t j = a->in_off[u]; j < a->in_off[u + 1]; j++) {
				sum = sat_add(sum, prev[a->in_src[j]]);
			}
			cur[u] = sum;
			alive |= sum != 0;
		}
		*stop = h;
		if (cur[t] > 0) {
			if (h > ORC_PATH_MAX) {
				return ORC_ERR_UNSUPPORTED;
			}
			r->ngroups++;
			r->count = sat_add(r->count, cur[t]);
			r->last = h;
		}
		if (!alive) {
			break;
		}
		if (r->ngroups < k && h > ORC_PATH_MAX) {
			return ORC_ERR_UNSUPPORTED; /* a longer group exists and is needed */
		}
	}
	if (count_only) {
		return ORC_OK;
	}
	if (max_paths == 0 && r->count == INT64_MAX) {
		return ORC_ERR_UNSUPPORTED;
	}
	for (int64_t h = 0; h <= r->last; h++) {
		const int64_t c = a->layer[h][t];
		const int64_t room = max_paths ? max_paths - r->npaths : c;
		const int64_t want = c < room ? c : room;
		if (want > 0) {
			int rc = enumerate(a, t, h, want);
			if (rc) {
				return rc;
			}
			r->npaths += want;
		}
	}
	r->complete = r->npaths == r->count;
	return ORC_OK;
}

/* ---- TRAIL, ACYCLIC, SIMPLE ---- */

static int round_add(orc_kg *a, int64_t r, int64_t x) {
	while (a->nrounds <= r) {
		vec *nr = (vec *)realloc(a->round_x, (size_t)(a->nrounds + 1) * sizeof(vec));
		if (!nr) {
			return ORC_ERR_ALLOC;
		}
		a->round_x = nr;
		memset(&a->round_x[a->nrounds], 0, sizeof(vec));
		a->nrounds++;
	}
	return vec_push(&a->round_x[r], x);
}

/* one spur search from u to t under the current stamps: *took = it had an admissible first edge, *x = its forward
 * expansions, *h = the spur's length (0: t not found), the spur in sp_vert / sp_pos */
static int spur(orc_kg *a, int64_t u, int64_t t, int *took, int64_t *x, int64_t *h) {
	const int64_t st = a->stamp;
	int64_t nq = 0;
	*took = 0;
	*x = 0;
	*h = 0;
	for (int64_t w = 0; w < a->n; w++) {
		a->lvl[w] = a->vban[w] == st ? -2 : -1; /* -2: banned, -1: unseen */
	}
	for (int64_t idx = a->v[u]; idx < a->v[u + 1]; idx++) {
		const int64_t w = a->e[idx];
		if (a->dban[idx] == st || a->eban[idx] == st || a->vban[w] == st) {
			continue;
		}
		*took = 1;
		if (a->lvl[w] == -1) {
			a->lvl[w] = 1;
			a->queue[nq++] = w;
		}
	}
	if (!*took) {
		return ORC_OK;
	}
	int64_t lv = 1;
	while (a->lvl[t] < 1 && nq > 0) {
		(*x)++;
		lv++;
		int64_t nn = 0;
		for (int64_t q = 0; q < nq; q++) {
			const int64_t r = a->queue[q];
			for (int64_t idx = a->v[r]; idx < a->v[r + 1]; idx++) {
				const int64_t w = a->e[idx];
				if (a->eban[idx] == st || a->lvl[w] != -1) {
					continue;
				}
				if (lv > ORC_PATH_MAX) {
					return ORC_ERR_UNSUPPORTED;
				}
				a->lvl[w] = lv;
				a->nextq[nn++] = w;
			}
		}
		int64_t *tmp = a->queue;
		a->queue = a->nextq;
		a->nextq = tmp;
		nq = nn;
	}
	if (a->lvl[t] < 1) {
		return ORC_OK;
	}
	const int64_t H = a->lvl[t];
	int64_t cur = t;
	a->sp_vert[H] = t;
	for (int64_t l = H; l >= 2; l--) {
		int64_t j = a->in_off[cur];
		while (a->lvl[a->in_src[j]] != l - 1 || a->eban[a->in_idx[j]] == st) {
			j++;
		}
		a->sp_pos[l - 1] = a->in_idx[j];
		cur = a->in_src[j];
		a->sp_vert[l - 1] = cur;
	}
	int64_t idx = a->v[u];
	while (a->e[idx] != cur || a->dban[idx] == st || a->eban[idx] == st) {
		idx++;
	}
	a->sp_pos[0] = idx;
	a->sp_vert[0] = u;
	*h = H;
	return ORC_OK;
}

static int grow(path **arr, int64_t *cap, int64_t need) {
	if (need <= *cap) {
		return ORC_OK;
	}
	int64_t c = *cap ? 2 * *cap : 16;
	while (c < need) {
		c *= 2;
	}
	path *d = (path *)realloc(*arr, (size_t)c * sizeof(path));
	if (!d) {
		return ORC_ERR_ALLOC;
	}
	*arr = d;
	*cap = c;
	return ORC_OK;
}

/* P's first j steps + the spur: into the sorted pool unless known (accepted or pooled) */
static int add_candidate(orc_kg *a, const path *P, int64_t j, int64_t sh) {
	path c;
	c.h = j + sh;
	c.dev = j;
	c.vert = (int64_t *)malloc((size_t)(c.h + 1) * sizeof(int64_t));
	c.pos = (int64_t *)malloc((size_t)(c.h + 1) * sizeof(int64_t));
	if (!c.vert || !c.pos) {
		path_free(&c);
		return ORC_ERR_ALLOC;
	}
	for (int64_t i = 0; i < j; i++) {
		c.vert[i] = P->vert[i];
		c.pos[i] = P->pos[i];
	}
	for (int64_t i = 0; i < sh; i++) {
		c.vert[j + i] = a->sp_vert[i];
		c.pos[j + i] = a->sp_pos[i];
	}
	c.vert[c.h] = a->sp_vert[sh];
	for (int64_t i = 0; i < a->nacc; i++) {
		if (!path_cmp(&a->acc[i], &c)) {
			path_free(&c);
			return ORC_OK;
		}
	}
	int64_t at = 0;
	while (at < a->npool && path_cmp(&a->pool[at], &c) < 0) {
		at++;
	}
	if (at < a->npool && !path_cmp(&a->pool[at], &c)) {
		path_free(&c);
		return ORC_OK;
	}
	if (grow(&a->pool, &a->cap_pool, a->npool + 1)) {
		path_free(&c);
		return ORC_ERR_ALLOC;
	}
	memmove(&a->pool[at + 1], &a->pool[at], (size_t)(a->npool - at) * sizeof(path));
	a->pool[at] = c;
	a->npool++;
	return ORC_OK;
}

static int run_spur(orc_kg *a, int64_t round, const path *P, int64_t j, int64_t t) {
	int took;
	int64_t x, sh;
	int rc = spur(a, P->vert[j], t, &took, &x, &sh);
	if (rc) {
		return rc;
	}
	if (took && (rc = round_add(a, round, x))) {
		return rc;
	}
	return sh ? add_candidate(a, P, j, sh) : ORC_OK;
}

/* one row of a path mode: its accepted paths in a->acc */
static int mode_row(orc_kg *a, int64_t s, int64_t t, int64_t k, int mode, int64_t max_paths, kg_row *r) {
	for (int64_t i = 0; i < a->nacc; i++) {
		path_free(&a->acc[i]);
	}
	for (int64_t i = 0; i < a->npool; i++) {
		path_free(&a->pool[i]);
	}
	a->nacc = a->npool = 0;
	memset(r, 0, sizeof(*r));
	r->last = -1;
	r->complete = 1;
	int rc;
	path root0 = {0, 0, NULL, NULL};
	int64_t root_vert = s;
	root0.vert = &root_vert;
	const int closed = s == t;
	for (int64_t round = 0;; round++) {
		if (round == 0 && closed) { /* [s], no search; with k = 1 every other path is past the group */
			if (grow(&a->acc, &a->cap_acc, 1)) {
				return ORC_ERR_ALLOC;
			}
			path p0 = {0, 0, (int64_t *)malloc(sizeof(int64_t)), (int64_t *)malloc(sizeof(int64_t))};
			if (!p0.vert || !p0.pos) {
				path_free(&p0);
				return ORC_ERR_ALLOC;
			}
			p0.vert[0] = s;
			a->acc[a->nacc++] = p0;
			r->ngroups = 1;
			if (k == 1) {
				break;
			}
			continue;
		}
		if (round == 0) {
			a->stamp++; /* no bans */
			if ((rc = run_spur(a, 0, &root0, 0, t))) {
				return rc;
			}
		} else {
			const path *P = &a->acc[a->nacc - 1];
			const int64_t L = P->h;
			int64_t j0 = P->dev, j1 = mode == ORC_TRAIL ? L : L - 1;
			if (mode == ORC_SIMPLE && closed && L == 0) {
				j0 = j1 = 0;
			}
			for (int64_t j = j0; j <= j1; j++) {
				const int64_t st = ++a->stamp;
				for (int64_t q = 0; q < a->nacc; q++) {
					const path *Q = &a->acc[q];
					if (Q->h > j && (j == 0 || !memcmp(Q->pos, P->pos, (size_t)j * sizeof(int64_t)))) {
						a->dban[Q->pos[j]] = st;
					}
				}
				for (int64_t i = 0; i <= j; i++) {
					if (mode == ORC_TRAIL) {
						if (i < j) {
							a->eban[P->pos[i]] = st;
						}
					} else if (!(closed && P->vert[i] == t)) {
						a->vban[P->vert[i]] = st;
					}
				}
				if ((rc = run_spur(a, round, P, j, t))) {
					return rc;
				}
			}
		}
		/* the pool's least path is the row's next path */
		if (a->npool == 0) {
			break;
		}
		if (r->ngroups == k && a->pool[0].h > a->acc[a->nacc - 1].h) {
			break;
		}
		if (max_paths && a->nacc == max_paths) {
			r->complete = 0;
			break;
		}
		if (a->pool[0].h > ORC_PATH_MAX) {
			return ORC_ERR_UNSUPPORTED;
		}
		if (a->nacc == 0 || a->pool[0].h > a->acc[a->nacc - 1].h) {
			r->ngroups++;
		}
		if (grow(&a->acc, &a->cap_acc, a->nacc + 1)) {
			return ORC_ERR_ALLOC;
		}
		a->acc[a->nacc++] = a->pool[0];
		memmove(&a->pool[0], &a->pool[1], (size_t)(a->npool - 1) * sizeof(path));
		a->npool--;
	}
	r->npaths = a->nacc;
	r->count = r->complete ? a->nacc : -1;
	r->last = a->nacc ? a->acc[a->nacc - 1].h : -1;
	for (int64_t q = 0; q < a->nacc; q++) {
		const path *P = &a->acc[q];
		if (vec_push(a->offsets, a->elems->size) || vec_push(a->elems, P->vert[0])) {
			return ORC_ERR_ALLOC;
		}
		for (int64_t x = 0; x < P->h; x++) {
			if (vec_push(a->elems, a->edge_ids[P->pos[x]]) || vec_push(a->elems, P->vert[x + 1])) {
				return ORC_ERR_ALLOC;
			}
		}
	}
	return ORC_OK;
}

/* Row i: out_count (N, -1 when unknown), out_ngroups, out_last (-1: none), out_complete, out_valid and out_npaths
 * paths from path out_first[i] on; path j is (*out_elems)[(*out_offsets)[j] .. (*out_offsets)[j + 1]).  count_only
 * (WALK): no lists.  lanes = 0: the header's rule.  stats (6 entries): batches, lanes, searches, levels, push_levels,
 * paths. */
int orc_shortest_k_groups(int64_t n, const int64_t *v, const int64_t *e, const int64_t *edge_ids, int64_t p,
                          const int64_t *src, const int64_t *dst, const uint8_t *src_valid, const uint8_t *dst_valid,
                          int64_t k, int32_t mode, int64_t max_paths, int32_t count_only, int64_t lanes,
                          int64_t *out_count, int64_t *out_ngroups, int64_t *out_last, uint8_t *out_complete,
                          int64_t *out_npaths, int64_t *out_first, uint8_t *out_valid, int64_t **out_offsets,
                          int64_t **out_elems, int64_t *stats) {
	if (n < 0 || p < 0 || k < 1 || max_paths < 0 || lanes < 0 || lanes % 64 || lanes > 512 || mode < ORC_WALK ||
	    mode > ORC_SIMPLE || (count_only && mode != ORC_WALK)) {
		return ORC_ERR_ARG;
	}
	for (int64_t i = 0; i < p; i++) {
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		if (src[i] < 0 || src[i] >= n || dst[i] < 0 || dst[i] >= n) {
			return ORC_ERR_RANGE;
		}
	}
	int rc = ORC_OK;
	const int64_t m = v[n];
	orc_kg a;
	memset(&a, 0, sizeof(a));
	a.n = n;
	a.m = m;
	a.v = v;
	a.e = e;
	a.edge_ids = edge_ids;
	vec elems = {0, 0, 0}, offsets = {0, 0, 0};
	a.elems = &elems;
	a.offsets = &offsets;
	a.in_off = (int64_t *)calloc((size_t)n + 2, sizeof(int64_t));
	a.in_src = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.in_idx = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.back = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.bq = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.wpath = (int64_t *)malloc((2 * (size_t)ORC_PATH_MAX + 4) * sizeof(int64_t));
	a.cursor = (int64_t *)malloc(((size_t)ORC_PATH_MAX + 3) * sizeof(int64_t));
	a.lvl = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.queue = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.nextq = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.vban = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
	a.eban = (int64_t *)calloc((size_t)m + 1, sizeof(int64_t));
	a.dban = (int64_t *)calloc((size_t)m + 1, sizeof(int64_t));
	a.sp_pos = (int64_t *)malloc(((size_t)n + 2) * sizeof(int64_t));
	a.sp_vert = (int64_t *)malloc(((size_t)n + 2) * sizeof(int64_t));
	int64_t *fill = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
	if (!a.in_off || !a.in_src || !a.in_idx || !a.back || !a.bq || !a.wpath || !a.cursor || !a.lvl || !a.queue ||
	    !a.nextq || !a.vban || !a.eban || !a.dban || !a.sp_pos || !a.sp_vert || !fill) {
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
	memset(stats, 0, 6 * sizeof(int64_t));
	int64_t searches = 0;
	for (int64_t i = 0; i < p; i++) {
		searches += !((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i]));
	}
	/* WALK's lane width: opts->lanes, or ks_lanes' rule over n_ab and the rows that take lanes */
	int64_t W = lanes;
	if (mode == ORC_WALK && !W) {
		int64_t n_ab = 0;
		for (int64_t u = 0; u < n; u++) {
			n_ab += a.in_off[u + 1] > a.in_off[u];
		}
		W = 512;
		while (W > 64 && 2 * (n_ab > 1 ? n_ab : 1) * W * 8 > ORC_BUDGET) {
			W >>= 1;
		}
		while (W > 64 && searches <= W / 2) {
			W >>= 1;
		}
	}
	int64_t lane = 0, batch_levels = 0, batch_push = 0;
	for (int64_t i = 0; i < p; i++) {
		out_count[i] = 0;
		out_ngroups[i] = 0;
		out_last[i] = -1;
		out_complete[i] = 1;
		out_npaths[i] = 0;
		out_first[i] = offsets.size;
		out_valid[i] = 0;
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		kg_row r;
		if (mode == ORC_WALK) {
			int64_t stop, ecc;
			if ((rc = walk_row(&a, src[i], dst[i], k, max_paths, count_only, &r, &stop, &ecc))) {
				goto done;
			}
			batch_levels = stop > batch_levels ? stop : batch_levels;
			batch_push = ecc + 1 > batch_push ? ecc + 1 : batch_push;
			if (++lane == W) { /* a full batch */
				lane = 0;
				stats[0]++;
				stats[3] += batch_levels;
				stats[4] += batch_push;
				batch_levels = batch_push = 0;
			}
		} else if ((rc = mode_row(&a, src[i], dst[i], k, mode, max_paths, &r))) {
			goto done;
		}
		out_count[i] = r.count;
		out_ngroups[i] = r.ngroups;
		out_last[i] = r.last;
		out_complete[i] = (uint8_t)r.complete;
		out_npaths[i] = r.npaths;
		out_valid[i] = count_only ? r.count > 0 : r.npaths > 0;
	}
	if (mode == ORC_WALK) {
		if (lane > 0) {
			stats[0]++;
			stats[3] += batch_levels;
			stats[4] += batch_push;
		}
		stats[1] = W;
		stats[2] = searches;
	} else { /* the rounds packed into batches */
		int64_t cap = lanes;
		if (!cap) {
			cap = 512;
			while (cap > 64 && (n > 1 ? n : 1) * cap * 2 > ORC_BUDGET) {
				cap >>= 1;
			}
		}
		stats[1] = lanes ? lanes : 64;
		for (int64_t r = 0; r < a.nrounds; r++) {
			const vec *x = &a.round_x[r];
			int64_t w = cap;
			while (!lanes && w > 64 && x->size <= w / 2) {
				w >>= 1;
			}
			stats[1] = w > stats[1] ? w : stats[1];
			stats[2] += x->size;
			for (int64_t b0 = 0; b0 < x->size; b0 += w) {
				int64_t mx = 0;
				for (int64_t l = b0; l < b0 + w && l < x->size; l++) {
					mx = x->data[l] > mx ? x->data[l] : mx;
				}
				stats[0]++;
				stats[3] += mx;
			}
		}
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
	for (int64_t i = 0; i < a.nacc; i++) {
		path_free(&a.acc[i]);
	}
	for (int64_t i = 0; i < a.npool; i++) {
		path_free(&a.pool[i]);
	}
	for (int64_t r = 0; r < a.nrounds; r++) {
		free(a.round_x[r].data);
	}
	free(a.round_x);
	free(a.acc);
	free(a.pool);
	free(offsets.data);
	free(elems.data);
	free(a.in_off);
	free(a.in_src);
	free(a.in_idx);
	free(a.back);
	free(a.bq);
	free(a.wpath);
	free(a.cursor);
	free(a.lvl);
	free(a.queue);
	free(a.nextq);
	free(a.vban);
	free(a.eban);
	free(a.dban);
	free(a.sp_pos);
	free(a.sp_vert);
	free(fill);
	return rc;
}

void orc_kgroups_free(void *x) {
	free(x);
}
