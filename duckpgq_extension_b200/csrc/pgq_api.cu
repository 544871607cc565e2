// pgq_api.cu -- the host-pointer entry points of the C ABI (include/duckpgq_b200.h): stage the
// DataChunk-style inputs in HBM, run the device drivers of pgq_bfs.cu, copy the results back.
// Reference call sites being replaced: IterativeLengthFunction (iterativelength.cpp:34-143) and
// ShortestPathFunction (shortest_path.cpp:43-207).
#include <cstdlib>
#include <cstring>

#include "pgq_internal.h"

static int check_call(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst) {
	if (!csr) {
		return pgq_fail(PGQ_ERR_INVALID_ID, "%s", pgq_status_text(PGQ_ERR_INVALID_ID));
	}
	if (p < 0 || (p > 0 && (!src || !dst))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null or negative argument");
	}
	if (p >= 0x7fffffffLL) {
		return pgq_fail(PGQ_ERR_RANGE, "too many pairs in one call");
	}
	if (!csr->finalized) {
		return pgq_fail(PGQ_ERR_NOT_INITIALIZED, "%s", pgq_status_text(PGQ_ERR_NOT_INITIALIZED));
	}
	return PGQ_OK;
}

// The rows of a host-column call on the device: src, dst and valid (NULL: every row) copied from the host, and the
// row outputs reserved
struct DeviceRows {
	const int64_t *src = nullptr, *dst = nullptr;
	const uint8_t *valid = nullptr;
	int64_t *len = nullptr; // (not reserved for shortestpath, which returns lists)
	uint8_t *out_valid = nullptr;
	int64_t h2d = 0; // bytes copied to the device
};

static int stage_rows(Workspace *ws, int64_t p, const int64_t *src, const int64_t *dst, const uint8_t *valid,
                      bool lengths, DeviceRows *d) {
	const size_t b8 = (size_t)p * sizeof(int64_t);
	PGQ_TRY(stage_column(ws, WS_IN_SRC, src, b8, (const void **)&d->src));
	PGQ_TRY(stage_column(ws, WS_IN_DST, dst, b8, (const void **)&d->dst));
	if (lengths) {
		PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LEN, b8, (void **)&d->len));
	}
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_VALID, (size_t)p, (void **)&d->out_valid));
	PGQ_TRY(stage_column(ws, WS_IN_VALID, valid, (size_t)p, (const void **)&d->valid));
	d->h2d = 2 * (int64_t)b8 + (valid ? p : 0);
	return PGQ_OK;
}

extern "C" int pgq_iterativelength_device(pgq_csr *csr, int64_t p, const int64_t *d_src, const int64_t *d_dst,
                                          const uint8_t *d_src_valid, const pgq_options *opts, int64_t *d_out_len,
                                          uint8_t *d_out_valid, void *stream, pgq_stats *stats) {
	PGQ_TRY(check_call(csr, p, d_src, d_dst));
	if (p > 0 && (!d_out_len || !d_out_valid)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	g.used = (cudaStream_t)stream;
	g.has_used = true;
	const int rc = pgq_bfs_lengths_device(csr, g.ws, p, d_src, d_dst, d_src_valid, opts, d_out_len, d_out_valid,
	                                      (cudaStream_t)stream, stats);
	g.settled = (rc == PGQ_OK); // (the driver has waited for the last level on its stream)
	return rc;
}

extern "C" int pgq_iterativelength(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                   const uint8_t *src_valid, const pgq_options *opts, int64_t *out_len,
                                   uint8_t *out_valid, pgq_stats *stats) {
	PGQ_TRY(check_call(csr, p, src, dst));
	if (p > 0 && (!out_len || !out_valid)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	if (p == 0) {
		if (stats) {
			memset(stats, 0, sizeof(*stats));
		}
		return PGQ_OK;
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	DeviceRows d;
	PGQ_TRY(stage_rows(ws, p, src, dst, src_valid, true, &d));
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	PGQ_TRY(pgq_bfs_lengths_device(csr, ws, p, d.src, d.dst, d.valid, opts, d.len, d.out_valid, s, &st));
	PGQ_CUDA(cudaMemcpyAsync(out_len, d.len, b8, cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaMemcpyAsync(out_valid, d.out_valid, (size_t)p, cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	g.settled = true;
	st.h2d_bytes += d.h2d;
	st.d2h_bytes += (int64_t)b8 + p;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_iterativelength_bidirectional(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                                 const uint8_t *src_valid, const uint8_t *dst_valid,
                                                 const pgq_options *opts, int64_t *out_len, uint8_t *out_valid,
                                                 pgq_stats *stats) {
	PGQ_TRY(check_call(csr, p, src, dst));
	if (p > 0 && (!out_len || !out_valid)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	DeviceRows d;
	std::vector<uint8_t> valid; // a row searches only when both of its ids are valid
	if (p > 0) {
		if (src_valid || dst_valid) {
			valid.resize((size_t)p);
			for (int64_t i = 0; i < p; i++) {
				valid[(size_t)i] = (!src_valid || src_valid[i]) && (!dst_valid || dst_valid[i]) ? 1 : 0;
			}
		}
		PGQ_TRY(stage_rows(ws, p, src, dst, valid.empty() ? nullptr : valid.data(), true, &d));
	}
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	PGQ_TRY(pgq_bfs_bidirectional_device(csr, ws, p, d.src, d.dst, d.valid, opts, d.len, d.out_valid, s, &st));
	if (p > 0) {
		PGQ_CUDA(cudaMemcpyAsync(out_len, d.len, b8, cudaMemcpyDeviceToHost, s));
		PGQ_CUDA(cudaMemcpyAsync(out_valid, d.out_valid, (size_t)p, cudaMemcpyDeviceToHost, s));
	}
	PGQ_CUDA(cudaStreamSynchronize(s));
	g.settled = true;
	st.h2d_bytes += d.h2d;
	st.d2h_bytes += p > 0 ? (int64_t)b8 + p : 0;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_reachability(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                const uint8_t *src_valid, const uint8_t *dst_valid, const pgq_options *opts, uint8_t *out,
                                uint8_t *out_valid, pgq_stats *stats) {
	PGQ_TRY(check_call(csr, p, src, dst));
	if (p > 0 && (!out || !out_valid)) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	const bool ref = opts && (opts->flags & PGQ_OPT_REFERENCE_BATCHING);
	// answered rows: both ids valid.  The searches: by default those rows; with the reference's batches every row with
	// a valid source, a NULL destination replaced by the source (the row keeps its lane and is answered NULL)
	std::vector<uint8_t> valid((size_t)p);
	std::vector<int64_t> search_dst;
	for (int64_t i = 0; i < p; i++) {
		const bool sv = !src_valid || src_valid[i], dv = !dst_valid || dst_valid[i];
		if ((sv && (src[i] < 0 || src[i] >= csr->n)) || (dv && (dst[i] < 0 || dst[i] >= csr->n))) {
			return pgq_fail(PGQ_ERR_RANGE, "source or destination rowid outside [0,%lld)", (long long)csr->n);
		}
		valid[(size_t)i] = sv && dv;
	}
	const uint8_t *h_sv = ref ? src_valid : (src_valid || dst_valid ? valid.data() : nullptr);
	const int64_t *h_dst = dst;
	if (ref && dst_valid) {
		search_dst.assign(dst, dst + p);
		for (int64_t i = 0; i < p; i++) {
			if (!dst_valid[i]) {
				search_dst[(size_t)i] = src[i];
			}
		}
		h_dst = search_dst.data();
	}
	if (p == 0) {
		if (stats) {
			memset(stats, 0, sizeof(*stats));
		}
		return PGQ_OK;
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	DeviceRows d;
	PGQ_TRY(stage_rows(ws, p, src, h_dst, h_sv, true, &d));
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	PGQ_TRY(pgq_bfs_reachability_device(csr, ws, p, d.src, d.dst, d.valid, src, h_sv, opts, d.len, d.out_valid, s,
	                                    &st));
	PGQ_CUDA(cudaMemcpyAsync(out, d.out_valid, (size_t)p, cudaMemcpyDeviceToHost, s));
	PGQ_CUDA(cudaStreamSynchronize(s));
	g.settled = true;
	for (int64_t i = 0; i < p; i++) {
		out[i] &= valid[(size_t)i];
		out_valid[i] = valid[(size_t)i];
	}
	st.h2d_bytes += d.h2d;
	st.d2h_bytes += p;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" int pgq_shortestpath(pgq_csr *csr, int64_t p, const int64_t *src, const int64_t *dst,
                                const uint8_t *src_valid, const pgq_options *opts, int64_t *out_offsets,
                                int64_t *out_lengths, uint8_t *out_valid, int64_t **out_elems, int64_t *out_total,
                                pgq_stats *stats) {
	PGQ_TRY(check_call(csr, p, src, dst));
	if (!out_elems || !out_total || (p > 0 && (!out_offsets || !out_lengths || !out_valid))) {
		return pgq_fail(PGQ_ERR_INVALID_ARG, "null output");
	}
	*out_elems = nullptr;
	*out_total = 0;
	if (p == 0) {
		if (stats) {
			memset(stats, 0, sizeof(*stats));
		}
		return PGQ_OK;
	}
	PGQ_CUDA(cudaSetDevice(csr->ctx->device));
	WsGuard g(csr->ctx);
	PGQ_TRY(pgq_ws_acquire(csr->ctx, &g.ws));
	Workspace *ws = g.ws;
	cudaStream_t s = ws->stream;
	int64_t *d_off, *d_lens;
	const size_t b8 = (size_t)p * sizeof(int64_t);
	DeviceRows d;
	PGQ_TRY(stage_rows(ws, p, src, dst, src_valid, false, &d));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_OFFSETS, b8, (void **)&d_off));
	PGQ_TRY(pgq_ws_reserve(ws, WS_OUT_LENGTHS, b8, (void **)&d_lens));
	pgq_stats st;
	memset(&st, 0, sizeof(st));
	int64_t *d_elems = nullptr;
	int64_t total = 0;
	// (d_elems points into the workspace)
	int rc = pgq_bfs_paths_device(csr, ws, p, d.src, d.dst, d.valid, opts, d_off, d_lens, d.out_valid, &d_elems, &total,
	                              s, &st);
	if (rc != PGQ_OK) {
		return rc;
	}
	int64_t *h_elems = (int64_t *)malloc((size_t)(total > 0 ? total : 1) * sizeof(int64_t));
	if (!h_elems) {
		return pgq_fail(PGQ_ERR_OOM, "host allocation of %lld path elements failed", (long long)total);
	}
	cudaError_t e = cudaSuccess;
	if (total > 0) {
		e = cudaMemcpyAsync(h_elems, d_elems, (size_t)total * sizeof(int64_t), cudaMemcpyDeviceToHost, s);
	}
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_offsets, d_off, b8, cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_lengths, d_lens, b8, cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaMemcpyAsync(out_valid, d.out_valid, (size_t)p, cudaMemcpyDeviceToHost, s);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	g.settled = (e == cudaSuccess);
	if (e != cudaSuccess) {
		cudaGetLastError();
		free(h_elems);
		return pgq_fail(PGQ_ERR_CUDA, "copying paths back failed: %s", cudaGetErrorString(e));
	}
	st.h2d_bytes += d.h2d;
	st.d2h_bytes += 2 * (int64_t)b8 + p + total * (int64_t)sizeof(int64_t);
	*out_elems = h_elems;
	*out_total = total;
	if (stats) {
		*stats = st;
	}
	return PGQ_OK;
}

extern "C" void pgq_free(void *p) {
	free(p);
}
