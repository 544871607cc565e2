/* pgq_oracle_bidir.c -- loop-for-loop restatement of IterativeLengthBidirectionalFunction
 * (reference src/core/functions/scalar/iterativelength_bidirectional.cpp:12-153) over int64 vertex ids.
 *
 * TEST INFRASTRUCTURE ONLY: the checker of pgq_iterativelength_bidirectional.  Lanes are 64 * k bits (k = 8 is the
 * reference's LANE_LIMIT of 512).  Deviations in undefined territory, as the device implements them: a NULL
 * destination gives NULL and takes no lane; an id outside [0, n) returns -2.
 * Counters: batches (turns of the outer while loop, l.84), iterations (calls of the level function, both sides) and
 * edges_traversed (trips of its inner edge loop, l.21-24, both sides). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;

/* one plain BFS level of one side (l.12-33): next = (OR over frontier v, edge v->t of visit[v] at t) & ~seen */
static int level(int64_t n, const int64_t *v, const int64_t *e, int k, u64 *seen, const u64 *visit, u64 *next,
                 int64_t *edges) {
	int change = 0;
	memset(next, 0, (size_t)n * k * sizeof(u64));
	for (int64_t x = 0; x < n; x++) {
		int any = 0;
		for (int i = 0; i < k; i++) {
			any |= visit[x * k + i] != 0;
		}
		if (!any) {
			continue;
		}
		for (int64_t p = v[x]; p < v[x + 1]; p++) {
			const int64_t t = e[p];
			for (int i = 0; i < k; i++) {
				next[t * k + i] |= visit[x * k + i];
			}
			(*edges)++;
		}
	}
	for (int64_t x = 0; x < n * k; x++) {
		next[x] &= ~seen[x];
		seen[x] |= next[x];
		change |= next[x] != 0;
	}
	return change;
}

int orc_iterativelengthbidirectional(int64_t n, const int64_t *v, const int64_t *e, int64_t p, const int64_t *src,
                                     const int64_t *dst, const uint8_t *src_valid, const uint8_t *dst_valid, int k,
                                     int64_t *out, uint8_t *out_valid, int64_t *batches, int64_t *iterations,
                                     int64_t *edges) {
	const int lanes = 64 * k;
	const size_t words = (size_t)(n > 0 ? n : 1) * k;
	for (int64_t i = 0; i < p; i++) {
		const int ok = (!src_valid || src_valid[i]) && (!dst_valid || dst_valid[i]);
		if (ok && src[i] != dst[i] && (src[i] < 0 || src[i] >= n || dst[i] < 0 || dst[i] >= n)) {
			return -2;
		}
	}
	/* [side][0] seen, [side][1] visit1, [side][2] visit2 */
	u64 *a[2][3];
	int64_t *lane_to_num = (int64_t *)malloc((size_t)lanes * sizeof(int64_t));
	int rc = lane_to_num ? 0 : -1;
	for (int s = 0; s < 2; s++) {
		for (int j = 0; j < 3; j++) {
			a[s][j] = (u64 *)calloc(words, sizeof(u64));
			if (!a[s][j]) {
				rc = -1;
			}
		}
	}
	*batches = *iterations = *edges = 0;
	int64_t started = 0;
	while (rc == 0 && started < p) { /* l.84 */
		(*batches)++;
		for (int s = 0; s < 2; s++) {
			memset(a[s][0], 0, words * sizeof(u64));
			memset(a[s][1], 0, words * sizeof(u64));
		}
		int64_t active = 0;
		for (int lane = 0; lane < lanes; lane++) { /* l.95-116 */
			lane_to_num[lane] = -1;
			while (started < p) {
				const int64_t i = started++;
				const int ok = (!src_valid || src_valid[i]) && (!dst_valid || dst_valid[i]);
				if (!ok) {
					out_valid[i] = 0;
					out[i] = -1;
				} else if (src[i] == dst[i]) {
					out_valid[i] = 1;
					out[i] = 0;
				} else {
					const u64 bit = 1ull << (lane & 63);
					a[0][1][src[i] * k + lane / 64] |= bit;
					a[1][1][dst[i] * k + lane / 64] |= bit;
					a[0][0][src[i] * k + lane / 64] |= bit;
					a[1][0][dst[i] * k + lane / 64] |= bit;
					lane_to_num[lane] = i;
					out_valid[i] = 0;
					out[i] = -1;
					active++;
					break;
				}
			}
		}
		for (int64_t iter = 0; active; iter++) { /* l.119-141 */
			const int s = (int)(iter & 1);
			const int from = (iter & 2) ? 2 : 1;
			(*iterations)++;
			if (!level(n, v, e, k, a[s][0], a[s][from], a[s][3 - from], edges)) {
				break;
			}
			for (int lane = 0; lane < lanes; lane++) {
				const int64_t num = lane_to_num[lane];
				if (num < 0) {
					continue;
				}
				int met = 0;
				for (int64_t x = 0; x < n && !met; x++) {
					met = ((a[0][0][x * k + lane / 64] & a[1][0][x * k + lane / 64]) >> (lane & 63)) & 1;
				}
				if (met) {
					out[num] = iter + 1;
					out_valid[num] = 1;
					lane_to_num[lane] = -1;
					active--;
				}
			}
		}
		/* lanes not met stay NULL (l.143-150) */
	}
	for (int s = 0; s < 2; s++) {
		for (int j = 0; j < 3; j++) {
			free(a[s][j]);
		}
	}
	free(lane_to_num);
	return rc;
}
