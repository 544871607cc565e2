/*
 * pgq_oracle_cheapest_k.c -- CPU restatement of cheapest_k_paths: the k cheapest paths of a row in the WALK, TRAIL,
 * ACYCLIC and SIMPLE path modes over a weighted CSR (SQL/PGQ's CHEAPEST k; no reference function).
 *
 * TEST INFRASTRUCTURE ONLY, like pgq_oracle.c: the checker of pgq_cheapest_k_paths.  Only tests/ and tools/ may build,
 * load or call this file; the product never links or falls back to it.
 *
 * Written from the definitions in include/duckpgq_b200.h alone, over the reference CSR layout (v offsets, e targets,
 * edge ids, weights as raw bits), one row at a time: Yen's algorithm with Lawler's rule, with one sequential
 * Bellman-Ford per spur search (its fixed point does not depend on the order of the relaxations), a BFS over the tight
 * edges it leaves, the same walk back, and a sorted array as the candidate pool.  The stats at a given lane width
 * simulate the rounds: every spur search that takes a lane is recorded with its round and its number of tight
 * expansions, and the rounds are then packed into batches, in (row, j) order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_ERR_ALLOC 1
#define ORC_ERR_ARG 2
#define ORC_ERR_RANGE 3
#define ORC_ERR_UNSUPPORTED 4

#define ORC_PATH_MAX 65533
#define ORC_LEVEL_MAX 65534
#define ORC_WALK 0
#define ORC_TRAIL 1
#define ORC_ACYCLIC 2
#define ORC_SIMPLE 3
#define ORC_BUDGET ((int64_t)2 << 30)
#define ORC_INF_I64 (INT64_MAX / 2)
#define ORC_INF_F64 (1.7976931348623157e308 / 2)

typedef struct {
	int64_t *data;
	int64_t size, cap;
} vec;

static int vec_push(vec *x, int64_t val) {
	if (x->size == x->cap) {
		int64_t cap = x->cap ? 2 * x->cap : 16;
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

static int f64_mode; /* the weights are doubles */

static double as_f64(int64_t b) {
	double d;
	memcpy(&d, &b, sizeof(d));
	return d;
}

static int64_t f64_bits(double d) {
	int64_t b;
	memcpy(&b, &d, sizeof(b));
	return b;
}

/* *r = c + w in the weight type's arithmetic; 0 when the sum is NaN or reaches the sentinel (tested before the
 * addition for BIGINT) */
static int sum(int64_t c, int64_t w, int64_t *r) {
	if (f64_mode) {
		const double x = as_f64(c) + as_f64(w);
		*r = f64_bits(x);
		return x < ORC_INF_F64;
	}
	if (!(w < ORC_INF_I64 - c)) {
		return 0;
	}
	*r = c + w;
	return 1;
}

static int cost_cmp(int64_t a, int64_t b) {
	if (f64_mode) {
		const double x = as_f64(a), y = as_f64(b);
		return x < y ? -1 : x > y ? 1 : 0;
	}
	return a < b ? -1 : a > b ? 1 : 0;
}

/* a path: h edges; vert[0..h] original vertex ids, pos[0..h) CSR positions (global), pc[0..h] prefix costs, dev */
typedef struct {
	int64_t h, dev;
	int64_t *vert, *pos, *pc;
} path;

static void path_free(path *p) {
	free(p->vert);
	free(p->pos);
	free(p->pc);
	p->vert = p->pos = p->pc = NULL;
}

/* the result's order: cost, h, then (parent, position) from t back to s */
static int path_cmp(const path *a, const path *b) {
	const int c = cost_cmp(a->pc[a->h], b->pc[b->h]);
	if (c) {
		return c;
	}
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
	const int64_t *v, *e, *w;
	int64_t *in_off, *in_src, *in_idx; /* in-lists in step order */
	int64_t *dist, *lvl, *queue, *nextq;
	int64_t *vban, *eban, *dban; /* stamps */
	int64_t stamp;
	int64_t *sp_pos, *sp_vert; /* the spur found, from u on */
	path *acc, *pool;
	int64_t nacc, npool, cap_acc, cap_pool;
	vec *round_x; /* per round: the tight expansions of each search that took a lane */
	int64_t nrounds;
} orc_ck;

static int round_add(orc_ck *a, int64_t r, int64_t x) {
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

/* the edge at position idx (to x) is tight from the cost c: c + w(idx) == d(x) as values, the sum below the sentinel */
static int tight(const orc_ck *a, int64_t c, int64_t idx, int64_t x) {
	int64_t r;
	return sum(c, a->w[idx], &r) && !cost_cmp(r, a->dist[x]);
}

/* first edge idx of u's adjacency (to x) is admissible under the current stamps */
static int first_ok(const orc_ck *a, int64_t idx, int64_t x) {
	const int64_t st = a->stamp;
	return a->dban[idx] != st && a->eban[idx] != st && a->vban[x] != st;
}

/* One spur search from u to t with root cost rc under the current stamps: *took = it had an admissible seed (and so
 * took a lane), *x = its tight expansions, *h = the spur's length (0: t not found), the spur in sp_vert / sp_pos */
static int spur(orc_ck *a, int64_t u, int64_t t, int64_t rc, int *took, int64_t *x, int64_t *h) {
	const int64_t st = a->stamp;
	const int64_t inf = f64_mode ? f64_bits(ORC_INF_F64) : ORC_INF_I64;
	*took = 0;
	*x = 0;
	*h = 0;
	for (int64_t y = 0; y < a->n; y++) {
		a->dist[y] = inf;
		a->lvl[y] = -1;
	}
	/* seeds, then sweeps to the fixed point */
	for (int64_t idx = a->v[u]; idx < a->v[u + 1]; idx++) {
		const int64_t y = a->e[idx];
		int64_t r;
		if (first_ok(a, idx, y) && sum(rc, a->w[idx], &r)) {
			*took = 1;
			if (cost_cmp(r, a->dist[y]) < 0) {
				a->dist[y] = r;
			}
		}
	}
	if (!*took) {
		return ORC_OK;
	}
	for (int changed = 1; changed;) {
		changed = 0;
		for (int64_t r0 = 0; r0 < a->n; r0++) {
			for (int64_t idx = a->v[r0]; idx < a->v[r0 + 1]; idx++) {
				const int64_t y = a->e[idx];
				int64_t r;
				if (a->eban[idx] == st || a->vban[y] == st || !sum(a->dist[r0], a->w[idx], &r)) {
					continue;
				}
				if (cost_cmp(r, a->dist[y]) < 0) {
					a->dist[y] = r;
					changed = 1;
				}
			}
		}
	}
	/* the tight BFS from the tight seeds (level 1) */
	int64_t nq = 0;
	for (int64_t idx = a->v[u]; idx < a->v[u + 1]; idx++) {
		const int64_t y = a->e[idx];
		if (first_ok(a, idx, y) && tight(a, rc, idx, y) && a->lvl[y] == -1) {
			a->lvl[y] = 1;
			a->queue[nq++] = y;
		}
	}
	int64_t lv = 1;
	while (a->lvl[t] < 1 && nq > 0) {
		if (lv + 1 > ORC_LEVEL_MAX) {
			return ORC_ERR_UNSUPPORTED;
		}
		(*x)++;
		int64_t nn = 0;
		for (int64_t q = 0; q < nq; q++) {
			const int64_t r0 = a->queue[q];
			for (int64_t idx = a->v[r0]; idx < a->v[r0 + 1]; idx++) {
				const int64_t y = a->e[idx];
				if (a->lvl[y] != -1 || a->eban[idx] == st || a->vban[y] == st || !tight(a, a->dist[r0], idx, y)) {
					continue;
				}
				a->lvl[y] = lv + 1;
				a->nextq[nn++] = y;
			}
		}
		lv++;
		int64_t *tmp = a->queue;
		a->queue = a->nextq;
		a->nextq = tmp;
		nq = nn;
	}
	if (a->lvl[t] < 1) {
		return ORC_OK;
	}
	/* the walk back */
	const int64_t H = a->lvl[t];
	int64_t cur = t;
	a->sp_vert[H] = t;
	for (int64_t l = H; l >= 2; l--) {
		int64_t j = a->in_off[cur];
		while (a->lvl[a->in_src[j]] != l - 1 || a->eban[a->in_idx[j]] == st ||
		       !tight(a, a->dist[a->in_src[j]], a->in_idx[j], cur)) {
			j++;
		}
		a->sp_pos[l - 1] = a->in_idx[j];
		cur = a->in_src[j];
		a->sp_vert[l - 1] = cur;
	}
	int64_t idx = a->v[u];
	while (a->e[idx] != cur || !first_ok(a, idx, cur) || !tight(a, rc, idx, cur)) {
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

/* R (P's first j steps) + the spur: into the pool unless known (in A or the pool) */
static int add_candidate(orc_ck *a, const path *P, int64_t j, int64_t sh) {
	path c;
	c.h = j + sh;
	c.dev = j;
	c.vert = (int64_t *)malloc((size_t)(c.h + 1) * sizeof(int64_t));
	c.pos = (int64_t *)malloc((size_t)(c.h + 1) * sizeof(int64_t));
	c.pc = (int64_t *)malloc((size_t)(c.h + 1) * sizeof(int64_t));
	if (!c.vert || !c.pos || !c.pc) {
		path_free(&c);
		return ORC_ERR_ALLOC;
	}
	for (int64_t i = 0; i < j; i++) {
		c.vert[i] = P->vert[i];
		c.pos[i] = P->pos[i];
	}
	for (int64_t i = 0; i <= j; i++) {
		c.pc[i] = P->pc[i];
	}
	for (int64_t i = 0; i < sh; i++) {
		c.vert[j + i] = a->sp_vert[i];
		c.pos[j + i] = a->sp_pos[i];
		sum(c.pc[j + i], a->w[a->sp_pos[i]], &c.pc[j + i + 1]); /* (a tight step: below the sentinel) */
	}
	c.vert[c.h] = a->sp_vert[sh];
	for (int64_t i = 0; i < a->nacc; i++) {
		if (!path_cmp(&a->acc[i], &c)) {
			path_free(&c);
			return ORC_OK;
		}
	}
	int64_t at = 0; /* the pool is sorted */
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

static int run_spur(orc_ck *a, int64_t round, const path *P, int64_t j, int64_t t) {
	int took;
	int64_t x, sh;
	int rc = spur(a, P->vert[j], t, P->pc[j], &took, &x, &sh);
	if (rc) {
		return rc;
	}
	if (took && (rc = round_add(a, round, x))) {
		return rc;
	}
	return sh ? add_candidate(a, P, j, sh) : ORC_OK;
}

/* one row: its accepted paths in a->acc */
static int one_row(orc_ck *a, int64_t s, int64_t t, int64_t k, int mode) {
	for (int64_t i = 0; i < a->nacc; i++) {
		path_free(&a->acc[i]);
	}
	for (int64_t i = 0; i < a->npool; i++) {
		path_free(&a->pool[i]);
	}
	a->nacc = a->npool = 0;
	int rc;
	int64_t root_vert = s, root_pc = 0;
	path root0 = {0, 0, &root_vert, NULL, &root_pc};
	const int closed = s == t;
	for (int64_t round = 0; a->nacc < k; round++) {
		if (round == 0 && closed) {
			if (grow(&a->acc, &a->cap_acc, 1)) {
				return ORC_ERR_ALLOC;
			}
			path p0 = {0, 0, (int64_t *)malloc(sizeof(int64_t)), (int64_t *)malloc(sizeof(int64_t)),
			           (int64_t *)malloc(sizeof(int64_t))};
			if (!p0.vert || !p0.pos || !p0.pc) {
				path_free(&p0);
				return ORC_ERR_ALLOC;
			}
			p0.vert[0] = s;
			p0.pc[0] = 0;
			a->acc[a->nacc++] = p0;
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
			int64_t j0 = P->dev, j1 = mode == ORC_TRAIL || mode == ORC_WALK ? L : L - 1;
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
					} else if (mode != ORC_WALK && !(closed && P->vert[i] == t)) {
						a->vban[P->vert[i]] = st;
					}
				}
				if ((rc = run_spur(a, round, P, j, t))) {
					return rc;
				}
			}
		}
		if (a->npool == 0) {
			break;
		}
		if (a->pool[0].h > ORC_PATH_MAX) {
			return ORC_ERR_UNSUPPORTED;
		}
		if (grow(&a->acc, &a->cap_acc, a->nacc + 1)) {
			return ORC_ERR_ALLOC;
		}
		a->acc[a->nacc++] = a->pool[0];
		memmove(&a->pool[0], &a->pool[1], (size_t)(a->npool - 1) * sizeof(path));
		a->npool--;
	}
	return ORC_OK;
}

/* Row i: out_valid, out_npaths paths from path out_first[i] on; path j is (*out_elems)[(*out_offsets)[j] ..
 * (*out_offsets)[j + 1]) with cost (*out_costs)[j] (raw bits).  w: the weights' raw bits in CSR position order,
 * is_f64: they are doubles.  lanes = 0: the header's rule over n.  stats (5 entries): batches, lanes, searches,
 * push_levels, paths. */
int orc_cheapest_k_paths(int64_t n, const int64_t *v, const int64_t *e, const int64_t *edge_ids, const int64_t *w,
                         int is_f64, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *src_valid,
                         const uint8_t *dst_valid, int64_t k, int32_t mode, int64_t lanes, int64_t *out_npaths,
                         int64_t *out_first, uint8_t *out_valid, int64_t **out_offsets, int64_t **out_elems,
                         int64_t **out_costs, int64_t *stats) {
	if (n < 0 || p < 0 || k < 1 || (lanes != 0 && lanes != 32 && lanes != 64 && lanes != 128 && lanes != 256) ||
	    (mode != ORC_WALK && mode != ORC_TRAIL && mode != ORC_ACYCLIC && mode != ORC_SIMPLE)) {
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
	const int64_t m = v[n];
	for (int64_t idx = 0; idx < m; idx++) {
		if (is_f64 ? as_f64(w[idx]) < 0 : w[idx] < 0) {
			return ORC_ERR_UNSUPPORTED;
		}
	}
	f64_mode = is_f64;
	int rc = ORC_OK;
	orc_ck a;
	memset(&a, 0, sizeof(a));
	a.n = n;
	a.m = m;
	a.v = v;
	a.e = e;
	a.w = w;
	vec elems = {0, 0, 0}, offsets = {0, 0, 0}, costs = {0, 0, 0};
	a.in_off = (int64_t *)calloc((size_t)n + 2, sizeof(int64_t));
	a.in_src = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.in_idx = (int64_t *)malloc(((size_t)m + 1) * sizeof(int64_t));
	a.dist = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.lvl = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.queue = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.nextq = (int64_t *)malloc(((size_t)n + 1) * sizeof(int64_t));
	a.vban = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
	a.eban = (int64_t *)calloc((size_t)m + 1, sizeof(int64_t));
	a.dban = (int64_t *)calloc((size_t)m + 1, sizeof(int64_t));
	a.sp_pos = (int64_t *)malloc(((size_t)n + 2) * sizeof(int64_t));
	a.sp_vert = (int64_t *)malloc(((size_t)n + 2) * sizeof(int64_t));
	int64_t *fill = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
	if (!a.in_off || !a.in_src || !a.in_idx || !a.dist || !a.lvl || !a.queue || !a.nextq || !a.vban || !a.eban ||
	    !a.dban || !a.sp_pos || !a.sp_vert || !fill) {
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
		out_npaths[i] = 0;
		out_first[i] = offsets.size;
		out_valid[i] = 0;
		if ((src_valid && !src_valid[i]) || (dst_valid && !dst_valid[i])) {
			continue;
		}
		if ((rc = one_row(&a, src[i], dst[i], k, mode))) {
			goto done;
		}
		out_npaths[i] = a.nacc;
		out_valid[i] = a.nacc > 0;
		for (int64_t q = 0; q < a.nacc; q++) {
			const path *P = &a.acc[q];
			if (vec_push(&offsets, elems.size) || vec_push(&elems, P->vert[0]) || vec_push(&costs, P->pc[P->h])) {
				rc = ORC_ERR_ALLOC;
				goto done;
			}
			for (int64_t x = 0; x < P->h; x++) {
				if (vec_push(&elems, edge_ids[P->pos[x]]) || vec_push(&elems, P->vert[x + 1])) {
					rc = ORC_ERR_ALLOC;
					goto done;
				}
			}
		}
	}
	/* the rounds packed into batches */
	int64_t cap = lanes;
	if (!cap) {
		cap = 256;
		while (cap > 32 && (n > 1 ? n : 1) * cap * 8 > ORC_BUDGET) {
			cap >>= 1;
		}
	}
	memset(stats, 0, 5 * sizeof(int64_t));
	stats[1] = lanes ? lanes : 32;
	for (int64_t r = 0; r < a.nrounds; r++) {
		const vec *x = &a.round_x[r];
		int64_t wl = cap;
		while (!lanes && wl > 32 && x->size <= wl / 2) {
			wl >>= 1;
		}
		stats[1] = wl > stats[1] ? wl : stats[1];
		stats[2] += x->size;
		for (int64_t b0 = 0; b0 < x->size; b0 += wl) {
			int64_t mx = 0;
			for (int64_t l = b0; l < b0 + wl && l < x->size; l++) {
				mx = x->data[l] > mx ? x->data[l] : mx;
			}
			stats[0]++;
			stats[3] += mx;
		}
	}
	stats[4] = offsets.size;
	if (vec_push(&offsets, elems.size) || vec_push(&costs, 0)) {
		rc = ORC_ERR_ALLOC;
		goto done;
	}
	*out_offsets = offsets.data;
	*out_elems = elems.data;
	*out_costs = costs.data;
	offsets.data = NULL;
	elems.data = NULL;
	costs.data = NULL;
done:
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
	free(costs.data);
	free(a.in_off);
	free(a.in_src);
	free(a.in_idx);
	free(a.dist);
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

void orc_cheapest_k_free(void *x) {
	free(x);
}
