/* pgq_oracle_reach.c -- loop-for-loop restatement of ReachabilityFunction (reference
 * src/core/functions/scalar/reachability.cpp:15-254) over int64 vertex ids, both traversals (is_variant).
 *
 * TEST INFRASTRUCTURE ONLY: the checker of pgq_reachability.  Lanes are the reference's LANE_LIMIT of 512.
 * The search runs over `input_size` vertices of the CSR (v, e), as the reference's bitsets do.
 * Two ways to start the next batch:
 *   restart = 1  the reference's: result_size += curr_batch_size (l.251), which counts the rows with a valid source
 *                only, so a NULL source makes the next batch start early and re-run rows (their results are written
 *                again).  A batch that finds no valid source would never end: the call returns -3 instead.
 *                A row's destination is read whatever its validity (the reference reads the byte under a NULL).
 *   restart = 0  the defined one (pgq_reachability with PGQ_OPT_REFERENCE_BATCHING): the next batch starts behind the
 *                last row InitialiseBfs looked at; a stretch without a valid source runs no batch; a NULL destination
 *                gives NULL.
 * out_valid[i] = 1 for every row whose result was written (rows with a NULL source never are, l.236-250).
 * An id that is read and lies outside [0, input_size), or input_size outside [0, n + 1], returns -2.
 * Counters: batches (turns of the outer while loop, l.194), levels (turns of the inner one, l.205), edges (trips of
 * the edge loops of whichever level function ran: with is_variant a vertex can be expanded twice in one level, so
 * this is not the algorithmic W there) and stale_starts (batches whose first level ran in mode 1: FindMode saw a
 * visit_list left over from an earlier batch, l.184,208). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
#define K 8 /* 512 lanes */
#define LANES (64 * K)

static int any(const u64 *x) {
	u64 a = 0;
	for (int i = 0; i < K; i++) {
		a |= x[i];
	}
	return a != 0;
}

typedef struct {
	int64_t *a;
	int64_t len, cap;
} list_t;

static int push(list_t *l, int64_t x) {
	if (l->len == l->cap) {
		int64_t cap = l->cap ? 2 * l->cap : 64;
		int64_t *a = (int64_t *)realloc(l->a, (size_t)cap * sizeof(int64_t));
		if (!a) {
			return -1;
		}
		l->a = a;
		l->cap = cap;
	}
	l->a[l->len++] = x;
	return 0;
}

/* the update half every level function shares (l.55-67 and friends) for vertex x: next &= ~seen; seen |= next */
static int update(int64_t x, u64 *seen, u64 *next) {
	for (int i = 0; i < K; i++) {
		next[x * K + i] &= ~seen[x * K + i];
		seen[x * K + i] |= next[x * K + i];
	}
	return any(next + x * K);
}

/* the push half: next[t] |= visit[x] along every out-edge of x */
static void expand(int64_t x, const int64_t *v, const int64_t *e, const u64 *visit, u64 *next, int64_t *edges) {
	for (int64_t p = v[x]; p < v[x + 1]; p++) {
		const int64_t t = e[p];
		for (int i = 0; i < K; i++) {
			next[t * K + i] |= visit[x * K + i];
		}
		(*edges)++;
	}
}

int orc_reachability(int64_t n, const int64_t *v, const int64_t *e, int64_t input_size, int64_t p, const int64_t *src,
                     const int64_t *dst, const uint8_t *src_valid, const uint8_t *dst_valid, int is_variant, int restart,
                     uint8_t *out, uint8_t *out_valid, int64_t *batches, int64_t *levels, int64_t *edges,
                     int64_t *stale_starts) {
	*batches = *levels = *edges = *stale_starts = 0;
	if (input_size < 0 || input_size > n + 1) {
		return -2;
	}
	for (int64_t i = 0; i < p; i++) {
		const int sv = !src_valid || src_valid[i], dv = !dst_valid || dst_valid[i];
		if ((sv && (src[i] < 0 || src[i] >= input_size)) ||
		    (sv && (dv || restart) && (dst[i] < 0 || dst[i] >= input_size))) {
			return -2;
		}
		out[i] = 0;
		out_valid[i] = 0;
	}
	const size_t words = (size_t)(input_size > 0 ? input_size : 1) * K;
	u64 *seen = (u64 *)calloc(words, sizeof(u64));
	u64 *visit = (u64 *)calloc(words, sizeof(u64));
	u64 *next = (u64 *)calloc(words, sizeof(u64));
	int16_t *lane_of = (int16_t *)malloc((size_t)(input_size > 0 ? input_size : 1) * sizeof(int16_t));
	uint8_t *inset = (uint8_t *)calloc((size_t)(input_size > 0 ? input_size : 1), 1);
	int64_t *brow = (int64_t *)malloc((size_t)(p > 0 ? p : 1) * sizeof(int64_t));
	list_t visit_list = {0, 0, 0}, lane_srcs = {0, 0, 0}, nset = {0, 0, 0};
	int rc = (seen && visit && next && lane_of && inset && brow) ? 0 : -1;
	for (int64_t x = 0; rc == 0 && x < input_size; x++) {
		lane_of[x] = -1;
	}
	const size_t visit_limit = (size_t)input_size / 2; /* VISIT_SIZE_DIVISOR */
	size_t num_nodes_to_visit = 0;
	int64_t result_size = 0;
	while (rc == 0 && result_size < p) { /* l.194 */
		memset(seen, 0, words * sizeof(u64));
		memset(visit, 0, words * sizeof(u64));
		memset(next, 0, words * sizeof(u64));
		/* InitialiseBfs, l.15-39 */
		int lanes = 0;
		int64_t cbs = 0, i = result_size;
		lane_srcs.len = 0;
		for (; i < p && lanes < LANES; i++) {
			if (src_valid && !src_valid[i]) {
				continue;
			}
			const int64_t s = src[i];
			if (lane_of[s] < 0) {
				lane_of[s] = (int16_t)lanes;
				seen[s * K + lanes / 64] |= 1ull << (lanes & 63);
				visit[s * K + lanes / 64] |= 1ull << (lanes & 63);
				lanes++;
				if (push(&lane_srcs, s)) {
					rc = -1;
				}
			}
			brow[cbs++] = i;
		}
		if (cbs == 0) {
			if (restart) {
				rc = -3; /* the reference loops forever here */
			}
			break;
		}
		(*batches)++;
		int mode = 0, exit_early = 0;
		for (int lvl = 0; rc == 0 && !exit_early; lvl++) { /* l.205-234 */
			exit_early = 1;
			(*levels)++;
			if (is_variant) {
				/* FindMode, l.154-163 */
				if (mode == 0 && visit_list.len > 0) {
					mode = 1;
				} else if (mode == 1 && (size_t)visit_list.len > visit_limit) {
					mode = 2;
				} else if (mode == 2 && num_nodes_to_visit < visit_limit) {
					mode = 0;
				}
				if (lvl == 0 && mode == 1) {
					(*stale_starts)++;
				}
				if (mode == 1) { /* BfsWithArrayVariant, l.129-152 */
					nset.len = 0;
					for (int64_t j = 0; j < visit_list.len; j++) {
						const int64_t x = visit_list.a[j];
						for (int64_t q = v[x]; q < v[x + 1]; q++) {
							const int64_t t = e[q];
							for (int w = 0; w < K; w++) {
								next[t * K + w] |= visit[x * K + w];
							}
							(*edges)++;
							if (!inset[t]) {
								inset[t] = 1;
								if (push(&nset, t)) {
									rc = -1;
								}
							}
						}
					}
					visit_list.len = 0;
					for (int64_t j = 0; j < nset.len; j++) {
						const int64_t x = nset.a[j];
						inset[x] = 0;
						if (update(x, seen, next)) {
							exit_early = 0;
							if (push(&visit_list, x)) {
								rc = -1;
							}
						}
					}
				} else { /* mode 0: BfsWithoutArrayVariant l.41-69; mode 2: BfsTempStateVariant l.97-127 */
					for (int64_t x = 0; x < input_size; x++) {
						if (any(visit + x * K)) {
							expand(x, v, e, visit, next, edges);
						}
					}
					size_t cnt = 0;
					for (int64_t x = 0; x < input_size; x++) {
						if (!any(next + x * K)) {
							continue;
						}
						if (update(x, seen, next)) {
							exit_early = 0;
							cnt++;
							if (mode == 0 && push(&visit_list, x)) {
								rc = -1;
							}
						}
					}
					if (mode == 2) {
						num_nodes_to_visit = cnt;
					}
				}
			} else { /* BfsWithoutArray, l.71-95 */
				for (int64_t x = 0; x < input_size; x++) {
					if (any(visit + x * K)) {
						expand(x, v, e, visit, next, edges);
					}
				}
				for (int64_t x = 0; x < input_size; x++) {
					if (any(next + x * K) && update(x, seen, next)) {
						exit_early = 0;
					}
				}
			}
			/* visit = visit_next; visit_next = 0 (l.230-233) */
			u64 *t = visit;
			visit = next;
			next = t;
			memset(next, 0, words * sizeof(u64));
		}
		/* l.236-250: result = seen[target][lane] && seen[source][lane] */
		for (int64_t j = 0; j < cbs; j++) {
			const int64_t r = brow[j];
			const int64_t s = src[r];
			const int lane = lane_of[s];
			if (!restart && dst_valid && !dst_valid[r]) {
				out[r] = 0;
				out_valid[r] = 0;
				continue;
			}
			const int64_t t = dst[r];
			out[r] = ((seen[t * K + lane / 64] >> (lane & 63)) & 1) && ((seen[s * K + lane / 64] >> (lane & 63)) & 1);
			out_valid[r] = 1;
		}
		for (int64_t j = 0; j < lane_srcs.len; j++) {
			lane_of[lane_srcs.a[j]] = -1;
		}
		result_size = restart ? result_size + cbs : i; /* l.251 / the defined start */
	}
	free(seen);
	free(visit);
	free(next);
	free(lane_of);
	free(inset);
	free(brow);
	free(visit_list.a);
	free(lane_srcs.a);
	free(nset.a);
	return rc;
}
