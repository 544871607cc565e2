// duckpgq_b200 -- the DuckDB-side shim of the H100 path-finding hot path.
//
// Loaded after the unmodified `duckpgq` extension, it re-registers -- same names, same argument types,
// so ExtensionLoader::RegisterFunction (ALTER_ON_CONFLICT) replaces the CPU callbacks -- the scalar
// functions of the hot path:
//
//   create_csr_vertex / create_csr_edge (3 overloads) / delete_csr   csr_creation.cpp:86-238, csr_deletion.cpp:10-29
//   iterativelength / iterativelength2 / shortestpath                iterativelength.cpp:148-152, shortest_path.cpp:212-217
//   iterativelengthbidirectional / reachability                      iterativelength_bidirectional.cpp:158-163,
//                                                                    reachability.cpp:259-264
//   cheapest_path_length                                             cheapest_path_length.cpp:162-166
//   local_clustering_coefficient / pagerank / weakly_connected_component (the reference's binds, device callbacks)
//                                                                    local_clustering_coefficient.cpp:14-83,
//                                                                    pagerank.cpp:14-120, weakly_connected_component.cpp:37-113
//
// The MATCH rewriter calls all of them BY NAME in the SQL it generates (match.cpp:476-487,657-671,
// compressed_sparse_row.cpp:132-251), so every SQL/PGQ query keeps the reference's parser, binder and
// rewriter and runs its CSR construction and its searches through the C ABI of libduckpgq_b200.so.
//
// CSR ownership (SURVEY.md section 8b): the host CSR object in DuckPGQState::csr_list stays the registry
// entry every reference function looks up.  Each DataChunk of create_csr_vertex / create_csr_edge is
// forwarded to the device build (pgq_csr_add_*; asynchronous pinned staging, no upload at query time).
// What happens to the HOST arrays is a mode (PGQ_B200_HOST_CSR):
//   skip   (default) the reference's scatter into the int64 host arrays is not run at all; the functions
//          of the reference that read the host CSR (get_csr_v / _e / _w / _ptr, and csr_get_w_type for a CSR
//          without a usable device build) are
//          wrapped: the wrapper first materialises the host arrays from the device copy (pgq_csr_download,
//          the reference's own layout), then calls the captured reference callback;
//   mirror the captured reference callback runs for every chunk as well (host and device CSR side by side).
// The device copy follows the host entry's lifetime: erased at QueryEnd when the id is in csr_to_delete
// (duckpgq_state.cpp:162-170), by delete_csr, or with the connection.
//
// Error texts, NULL handling, csr_to_delete bookkeeping: as the reference, line by line (cited below).
#define DUCKDB_EXTENSION_MAIN

#include "duckpgq_b200_extension.hpp"

#include "duckdb/catalog/catalog_entry/scalar_function_catalog_entry.hpp"
#include "duckdb/catalog/catalog_entry/table_function_catalog_entry.hpp"
#include "duckdb/common/string_util.hpp"
#include "duckdb/common/vector/flat_vector.hpp"
#include "duckdb/common/vector/list_vector.hpp"
#include "duckdb/execution/expression_executor.hpp"
#include "duckdb/function/scalar_function.hpp"
#include "duckdb/function/table_function.hpp"
#include "duckdb/main/client_context.hpp"
#include "duckdb/main/client_context_state.hpp"
#include "duckdb/main/extension/extension_loader.hpp"
#include "duckdb/parser/parsed_data/create_table_function_info.hpp"
#include "duckdb/planner/expression/bound_function_expression.hpp"

#include "duckpgq/core/functions/function_data/cheapest_path_length_function_data.hpp"
#include "duckpgq/core/functions/function_data/iterative_length_function_data.hpp"
#include "duckpgq/core/functions/function_data/local_clustering_coefficient_function_data.hpp"
#include "duckpgq/core/functions/function_data/pagerank_function_data.hpp"
#include "duckpgq/core/functions/function_data/weakly_connected_component_function_data.hpp"
#include "duckpgq/core/utils/compressed_sparse_row.hpp"
#include "duckpgq/core/utils/duckpgq_utils.hpp"

#include "duckpgq_b200.h"

#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace duckdb {

// ---- process-wide device context ----------------------------------------------------------------
static std::mutex g_ctx_lock;
static pgq_ctx *g_ctx = nullptr;
static std::atomic<int64_t> g_calls_cheapest_path {0};
static std::atomic<int64_t> g_calls_path_count {0};
static std::atomic<int64_t> g_calls_cheapest_count {0};
static std::atomic<int64_t> g_calls_all_cheapest {0};
static std::atomic<int64_t> g_calls_cheapest_k {0};
static std::atomic<int64_t> g_calls_all_shortest {0};
static std::atomic<int64_t> g_calls_shortest_k {0};
static std::atomic<int64_t> g_calls_shortest_k_mode {0};
static std::atomic<int64_t> g_calls_shortest_k_groups {0};
static std::atomic<int64_t> g_calls_shortest_k_groups_count {0};
static std::atomic<int64_t> g_calls_lengths {0}, g_calls_paths {0}, g_calls_cheapest {0}, g_pairs {0}, g_uploads {0},
    g_device_builds {0}, g_chunks {0}, g_materialized {0}, g_calls_lcc {0}, g_calls_pagerank {0}, g_calls_wcc {0},
    g_calls_bidirectional {0}, g_calls_w_type {0}, g_calls_reachability {0};

[[noreturn]] static void ThrowStatus(int status) {
	string msg = pgq_last_error();
	switch (status) {
	case PGQ_ERR_CONSTRAINT:
	case PGQ_ERR_INVALID_ID:
	case PGQ_ERR_NOT_INITIALIZED:
		throw ConstraintException(pgq_status_text(status));
	case PGQ_ERR_INVALID_ARG:
	case PGQ_ERR_RANGE:
		throw InvalidInputException("duckpgq_b200: " + msg);
	case PGQ_ERR_OOM:
		throw OutOfMemoryException("duckpgq_b200: " + msg);
	default:
		throw IOException("duckpgq_b200: " + msg);
	}
}

static vector<int> DeviceList();

static pgq_ctx *DeviceContext() {
	std::lock_guard<std::mutex> guard(g_ctx_lock);
	if (!g_ctx) {
		int device = DeviceList()[0];
		int st = pgq_ctx_create(device, &g_ctx);
		if (st != PGQ_OK) {
			g_ctx = nullptr;
			ThrowStatus(st); // no CPU fallback: a missing GPU is an error
		}
	}
	return g_ctx;
}

static bool MirrorHostCsr() {
	const char *env = std::getenv("PGQ_B200_HOST_CSR");
	return env && std::strcmp(env, "mirror") == 0;
}

// ---- per-connection registry of device CSRs -------------------------------------------------------
struct DeviceCsr {
	pgq_csr *csr = nullptr;
	int64_t v_size = 0;
	string error;       // a chunk failed: the device copy is unusable (path functions fall back to an upload)
	bool materialized = false; // the host arrays hold this CSR
	bool finalized = false;    // the device build has been completed (no further chunks can be added)
	bool edges_started = false; // create_csr_edge chunks have arrived (all create_csr_vertex chunks come first)
	pgq_multi_csr *multi = nullptr; // replicas on the other GPUs of PGQ_B200_DEVICES (made on first use)
};

static void FreeDeviceCsr(DeviceCsr &entry) {
	pgq_multi_csr_free(entry.multi); // (replicas first: they were cloned from the primary)
	entry.multi = nullptr;
	pgq_csr_free(entry.csr);
	entry.csr = nullptr;
}

// PGQ_B200_DEVICES=0,1,2,3: the GPUs one connection may fan a DataChunk's searches out over (the first one is
// where the CSR is built).  Default: the single device PGQ_B200_DEVICE (or 0).
static vector<int> DeviceList() {
	vector<int> devices;
	if (const char *env = std::getenv("PGQ_B200_DEVICES")) {
		string text = env;
		size_t pos = 0;
		while (pos < text.size()) {
			size_t comma = text.find(',', pos);
			if (comma == string::npos) {
				comma = text.size();
			}
			if (comma > pos) {
				devices.push_back(std::atoi(text.substr(pos, comma - pos).c_str()));
			}
			pos = comma + 1;
		}
	}
	if (devices.empty()) {
		const char *env = std::getenv("PGQ_B200_DEVICE");
		devices.push_back(env ? std::atoi(env) : 0);
	}
	return devices;
}

class DuckPGQB200State : public ClientContextState {
public:
	~DuckPGQB200State() override {
		std::lock_guard<std::mutex> guard(lock);
		for (auto &entry : by_id) {
			FreeDeviceCsr(entry.second);
		}
		for (auto &entry : uploaded) {
			pgq_csr_free(entry.second);
		}
	}

	// The reference erases csr_to_delete at QueryEnd (duckpgq_state.cpp:162-170); the device copies go with them.
	// (The two states' QueryEnd callbacks run in unspecified order: an id is gone if it is marked OR already erased.)
	void QueryEnd(ClientContext &context) override {
		auto pgq_state = context.registered_state->Get<DuckPGQState>("duckpgq");
		std::lock_guard<std::mutex> guard(lock);
		for (auto it = by_id.begin(); it != by_id.end();) {
			bool gone = !pgq_state || pgq_state->csr_to_delete.count(it->first) ||
			            pgq_state->csr_list.find(it->first) == pgq_state->csr_list.end();
			if (gone) {
				FreeDeviceCsr(it->second);
				it = by_id.erase(it);
			} else {
				++it;
			}
		}
		for (auto &entry : uploaded) { // uploads are per statement: the host pointer may be reused
			pgq_csr_free(entry.second);
		}
		uploaded.clear();
	}

	// create_csr_vertex: the entry every later chunk of this id is forwarded to (CsrInitializeVertex,
	// csr_creation.cpp:14-41: idempotent under the lock)
	DeviceCsr &Building(int32_t id, int64_t v_size, bool vertex_chunk, bool *fresh = nullptr) {
		std::lock_guard<std::mutex> guard(lock);
		auto it = by_id.find(id);
		if (it != by_id.end() && vertex_chunk &&
		    (it->second.finalized || it->second.edges_started || it->second.v_size != v_size)) {
			// a create_csr_vertex chunk for an id whose edges have already arrived: a NEW CSR is being built under an
			// id that was never deleted (test/sql/scalar/get_csr_w_type.test does this): start over
			FreeDeviceCsr(it->second);
			by_id.erase(it);
			it = by_id.end();
		}
		if (fresh) {
			*fresh = it == by_id.end();
		}
		if (it == by_id.end()) {
			DeviceCsr entry;
			entry.v_size = v_size;
			int st = pgq_csr_create(DeviceContext(), v_size, &entry.csr);
			if (st != PGQ_OK) {
				ThrowStatus(st);
			}
			g_device_builds++;
			it = by_id.emplace(id, entry).first;
		}
		if (!vertex_chunk) {
			it->second.edges_started = true;
		}
		return it->second;
	}

	DeviceCsr *Find(int32_t id) {
		std::lock_guard<std::mutex> guard(lock);
		auto it = by_id.find(id);
		return it == by_id.end() ? nullptr : &it->second;
	}

	void Drop(int32_t id) {
		std::lock_guard<std::mutex> guard(lock);
		auto it = by_id.find(id);
		if (it != by_id.end()) {
			FreeDeviceCsr(it->second);
			by_id.erase(it);
		}
	}

	// The multi-GPU group of a device-built CSR (PGQ_B200_DEVICES lists more than one GPU), nullptr otherwise.
	pgq_multi_csr *MultiFor(pgq_csr *csr) {
		vector<int> devices = DeviceList();
		if (devices.size() < 2) {
			return nullptr;
		}
		std::lock_guard<std::mutex> guard(lock);
		for (auto &kv : by_id) {
			if (kv.second.csr != csr) {
				continue;
			}
			if (!kv.second.multi) {
				int st = pgq_multi_csr_create(csr, devices.data(), static_cast<int>(devices.size()), &kv.second.multi);
				if (st != PGQ_OK) {
					ThrowStatus(st);
				}
			}
			return kv.second.multi;
		}
		return nullptr; // (an uploaded CSR: single device)
	}

	// The device CSR a path function runs on: the one built from the create_csr_* chunks (finalised on first
	// use), else -- the CSR was created before this extension was loaded, or its device build failed while the
	// host arrays exist -- an upload of the host CSR, with its weights when it has them.
	pgq_csr *ForPathFunction(int32_t id, CSR &host, int64_t v_size) {
		if (auto entry = Find(id)) {
			if (entry->error.empty()) {
				int st = pgq_csr_finalize(entry->csr); // idempotent, serialised inside
				if (st == PGQ_OK) {
					entry->finalized = true;
					return entry->csr;
				}
				std::lock_guard<std::mutex> guard(lock);
				entry->error = pgq_last_error();
			}
			if (!host.initialized_e) {
				throw InvalidInputException("duckpgq_b200: device CSR build failed: " + entry->error);
			}
		}
		if (!host.initialized_e && host.e.empty() && Find(id) == nullptr && v_size > 0) {
			// vertices only (test/sql/path_finding/edgeless_graph.test): nothing to upload but the offsets
		}
		std::lock_guard<std::mutex> guard(lock);
		auto it = uploaded.find(&host);
		if (it != uploaded.end()) {
			return it->second;
		}
		auto *v = reinterpret_cast<int64_t *>(host.v); // as iterativelength.cpp:53
		// v has v_size + 2 entries; v[v_size] is the number of edges actually scattered (the undirected
		// CSR over-allocates e twofold, compressed_sparse_row.cpp:208-223)
		if (v_size < 0 || static_cast<idx_t>(v_size) + 2 > host.vsize) {
			throw InvalidInputException("duckpgq_b200: v_size does not match the CSR");
		}
		int64_t m = v[v_size];
		if (m < 0 || static_cast<idx_t>(m) > host.e.size()) {
			throw InvalidInputException("duckpgq_b200: CSR offsets exceed the edge array");
		}
		const int64_t *edge_ids = host.edge_ids.size() >= static_cast<idx_t>(m) ? host.edge_ids.data() : nullptr;
		pgq_csr *device = nullptr;
		int st;
		if (host.initialized_w && !(host.w.empty() && host.w_double.empty())) {
			// the weights of create_csr_edge's 8-argument overloads, told apart as csr_get_w_type does
			const bool f64 = host.w.empty();
			if ((f64 ? host.w_double.size() : host.w.size()) < static_cast<idx_t>(m)) {
				throw InvalidInputException("duckpgq_b200: CSR weights do not cover the edge array");
			}
			st = pgq_csr_upload_weighted(DeviceContext(), v_size, m, v, host.e.data(), edge_ids,
			                             f64 ? nullptr : host.w.data(), f64 ? host.w_double.data() : nullptr, &device);
		} else {
			st = pgq_csr_upload(DeviceContext(), v_size, m, v, host.e.data(), edge_ids, &device);
		}
		if (st != PGQ_OK) {
			ThrowStatus(st);
		}
		uploaded[&host] = device;
		g_uploads++;
		return device;
	}

	// Fills the host arrays of every CSR that so far exists on the device only (mode `skip`), in the reference's
	// own layout, so that a reference function can read them.
	void MaterialiseHost(DuckPGQState &pgq_state) {
		std::lock_guard<std::mutex> guard(lock);
		for (auto &kv : by_id) {
			DeviceCsr &entry = kv.second;
			auto host_it = pgq_state.csr_list.find(kv.first);
			if (entry.materialized || host_it == pgq_state.csr_list.end() || !entry.error.empty()) {
				continue;
			}
			CSR &host = *host_it->second;
			if (host.initialized_e) { // mirror mode, or already filled
				entry.materialized = true;
				continue;
			}
			int st = pgq_csr_finalize(entry.csr);
			int64_t n = 0, m = 0;
			if (st == PGQ_OK) {
				entry.finalized = true;
				st = pgq_csr_info(entry.csr, &n, &m, nullptr);
			}
			if (st != PGQ_OK) {
				ThrowStatus(st);
			}
			if (static_cast<idx_t>(n) + 2 != host.vsize) {
				throw InvalidInputException("duckpgq_b200: host and device CSR disagree on the vertex count");
			}
			host.e.resize(static_cast<idx_t>(m), 0); // CsrInitializeEdge, csr_creation.cpp:43-61
			host.edge_ids.resize(static_cast<idx_t>(m), 0);
			st = pgq_csr_download(entry.csr, reinterpret_cast<int64_t *>(host.v), host.e.data(), host.edge_ids.data());
			if (st != PGQ_OK) {
				ThrowStatus(st);
			}
			host.initialized_e = true;
			int wt = 0;
			pgq_csr_weight_type(entry.csr, &wt);
			if (wt != 0 && m > 0) { // CsrInitializeWeight, csr_creation.cpp:63-84
				void *dst;
				if (wt == 1) {
					host.w.resize(static_cast<idx_t>(m), 0);
					dst = host.w.data();
				} else {
					host.w_double.resize(static_cast<idx_t>(m), 0);
					dst = host.w_double.data();
				}
				st = pgq_csr_download_weights(entry.csr, dst);
				if (st != PGQ_OK) {
					ThrowStatus(st);
				}
				host.initialized_w = true;
			}
			entry.materialized = true;
			g_materialized++;
		}
	}

private:
	std::mutex lock;
	std::unordered_map<int32_t, DeviceCsr> by_id;
	std::unordered_map<CSR *, pgq_csr *> uploaded;
};

static shared_ptr<DuckPGQB200State> GetB200State(ClientContext &context) {
	return context.registered_state->GetOrCreate<DuckPGQB200State>("duckpgq_b200");
}

// ---- DataChunk column access ----------------------------------------------------------------------
// A BIGINT / DOUBLE column as a contiguous host array: the vector's own buffer when it is flat and NULL-free,
// a copy otherwise (`valid` then tells which rows to keep).
template <class T>
struct Column {
	const T *data = nullptr;
	vector<T> copy;
	UnifiedVectorFormat format;
	bool all_valid = true;

	Column(Vector &vec, idx_t count) {
		vec.ToUnifiedFormat(format);
		auto raw = reinterpret_cast<const T *>(format.data);
		bool identity = !format.sel->IsSet();
		all_valid = format.validity.CannotHaveNull();
		if (identity && all_valid) {
			data = raw;
			return;
		}
		copy.resize(count);
		for (idx_t i = 0; i < count; i++) {
			auto pos = format.sel->get_index(i);
			copy[i] = format.validity.RowIsValid(pos) ? raw[pos] : T();
		}
		data = copy.data();
	}
	bool RowIsValid(idx_t i) const {
		return all_valid || format.validity.RowIsValid(format.sel->get_index(i));
	}
};

// Flattens (src, dst) of a path-function DataChunk into contiguous host columns for the C ABI.
struct PairColumns {
	vector<int64_t> src, dst;
	vector<uint8_t> valid;

	PairColumns(DataChunk &args) {
		UnifiedVectorFormat vsrc, vdst;
		args.data[2].ToUnifiedFormat(vsrc);
		args.data[3].ToUnifiedFormat(vdst);
		auto src_data = reinterpret_cast<const int64_t *>(vsrc.data);
		auto dst_data = reinterpret_cast<const int64_t *>(vdst.data);
		idx_t count = args.size();
		src.resize(count);
		dst.resize(count);
		valid.resize(count);
		for (idx_t i = 0; i < count; i++) {
			auto src_pos = vsrc.sel->get_index(i);
			auto dst_pos = vdst.sel->get_index(i);
			// NULL source -> NULL result (iterativelength.cpp:99-101).  The reference never looks at the
			// validity of dst and would read an unspecified value; here a NULL destination is a NULL result.
			bool ok = vsrc.validity.RowIsValid(src_pos) && vdst.validity.RowIsValid(dst_pos);
			valid[i] = ok ? 1 : 0;
			src[i] = ok ? src_data[src_pos] : 0;
			dst[i] = ok ? dst_data[dst_pos] : 0;
		}
	}
};

static pgq_options OptionsFromEnv() {
	pgq_options opts;
	memset(&opts, 0, sizeof(opts));
	if (const char *env = std::getenv("PGQ_B200_LANES")) {
		opts.lanes = std::atoi(env);
	}
	if (const char *env = std::getenv("PGQ_B200_DIRECTION")) {
		opts.direction = std::atoi(env);
	}
	if (const char *env = std::getenv("PGQ_B200_FLAGS")) {
		opts.flags = std::atoi(env);
	}
	return opts;
}

// ---- create_csr_vertex ----------------------------------------------------------------------------------
static void CreateCsrVertexB200(const scalar_function_t &reference, DataChunk &args, ExpressionState &state,
                                Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CSRFunctionData>();
	// host side: the registry entry + v[dense_id + 2] = cnt (csr_creation.cpp:86-110) -- always the reference's
	// own callback: n + 2 counters, and every reference function finds the CSR it expects in csr_list
	reference(args, state, result);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	idx_t count = args.size();
	bool fresh = false;
	auto &entry = GetB200State(info.context)->Building(info.id, v_size, true, &fresh);
	if (fresh && !MirrorHostCsr()) {
		// the host arrays (if an earlier CSR of this id left any) no longer describe this CSR: they are filled
		// from the device copy when a reference function asks for them (MaterialiseHost)
		auto duckpgq_state = GetDuckPGQState(info.context);
		auto host = duckpgq_state->csr_list.find(info.id);
		if (host != duckpgq_state->csr_list.end()) {
			host->second->initialized_e = false;
			host->second->initialized_w = false;
			host->second->e.clear();
			host->second->edge_ids.clear();
			host->second->w.clear();
			host->second->w_double.clear();
		}
	}
	Column<int64_t> dense_id(args.data[2], count), cnt(args.data[3], count);
	if (!dense_id.all_valid || !cnt.all_valid) {
		return; // (BinaryExecutor skips NULL rows, csr_creation.cpp:103-109: nothing to forward for them)
	}
	int st = pgq_csr_add_vertex_counts(entry.csr, static_cast<int64_t>(count), dense_id.data, cnt.data, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_chunks++;
}

// ---- create_csr_edge (no weight / BIGINT weight / DOUBLE weight) -------------------------------------------
static void CreateCsrEdgeB200(const scalar_function_t &reference, DataChunk &args, ExpressionState &state,
                              Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CSRFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context, true);
	auto b200 = GetB200State(info.context);

	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	int64_t edge_size = args.data[2].GetValue(0).GetValue<int64_t>();
	int64_t edge_size_count = args.data[3].GetValue(0).GetValue<int64_t>();
	if (edge_size != edge_size_count) { // csr_creation.cpp:121-125
		b200->Drop(info.id);
		duckpgq_state->csr_to_delete.insert(info.id);
		throw ConstraintException("Non-existent/non-unique vertices detected. Make sure all "
		                          "vertices referred by edge tables exist and are unique for path-finding queries.");
	}
	const bool weighted = info.weight_type != LogicalType::SQLNULL;
	const bool mirror = MirrorHostCsr();
	idx_t count = args.size();
	if (mirror) {
		reference(args, state, result); // the reference's scatter into the int64 host arrays
	}
	Column<int64_t> src(args.data[4], count), dst(args.data[5], count), edge_id(args.data[6], count);
	bool is_double = false;
	unique_ptr<Column<int64_t>> w_int;
	unique_ptr<Column<double>> w_double;
	if (weighted) {
		is_double = args.data[7].GetType().InternalType() == PhysicalType::DOUBLE;
		if (is_double) {
			w_double = make_uniq<Column<double>>(args.data[7], count);
		} else {
			w_int = make_uniq<Column<int64_t>>(args.data[7], count);
		}
	}
	bool all_valid = src.all_valid && dst.all_valid && edge_id.all_valid &&
	                 (!weighted || (is_double ? w_double->all_valid : w_int->all_valid));
	if (!mirror) {
		// result = 1 per row, or (int32) weight; rows with a NULL are NULL and skipped (csr_creation.cpp:129-196)
		result.SetVectorType(VectorType::FLAT_VECTOR);
		auto result_data = FlatVector::GetDataMutable<int32_t>(result);
		auto &result_validity = FlatVector::ValidityMutable(result);
		for (idx_t i = 0; i < count; i++) {
			bool ok = all_valid || (src.RowIsValid(i) && dst.RowIsValid(i) && edge_id.RowIsValid(i) &&
			                        (!weighted || (is_double ? w_double->RowIsValid(i) : w_int->RowIsValid(i))));
			if (!ok) {
				result_validity.SetInvalid(i);
				continue;
			}
			result_data[i] = !weighted ? 1
			                 : is_double ? static_cast<int32_t>(w_double->data[i])
			                             : static_cast<int32_t>(w_int->data[i]);
		}
	}
	auto &entry = b200->Building(info.id, v_size, false);
	const int64_t *p_src = src.data, *p_dst = dst.data, *p_eid = edge_id.data;
	const int64_t *p_wi = weighted && !is_double ? w_int->data : nullptr;
	const double *p_wd = weighted && is_double ? w_double->data : nullptr;
	vector<int64_t> c_src, c_dst, c_eid, c_wi;
	vector<double> c_wd;
	int64_t rows = static_cast<int64_t>(count);
	if (!all_valid) { // compact the rows without a NULL (the reference skips the others)
		for (idx_t i = 0; i < count; i++) {
			bool ok = src.RowIsValid(i) && dst.RowIsValid(i) && edge_id.RowIsValid(i) &&
			          (!weighted || (is_double ? w_double->RowIsValid(i) : w_int->RowIsValid(i)));
			if (!ok) {
				continue;
			}
			c_src.push_back(src.data[i]);
			c_dst.push_back(dst.data[i]);
			c_eid.push_back(edge_id.data[i]);
			if (p_wi) {
				c_wi.push_back(w_int->data[i]);
			}
			if (p_wd) {
				c_wd.push_back(w_double->data[i]);
			}
		}
		rows = static_cast<int64_t>(c_src.size());
		p_src = c_src.data();
		p_dst = c_dst.data();
		p_eid = c_eid.data();
		p_wi = p_wi ? c_wi.data() : nullptr;
		p_wd = p_wd ? c_wd.data() : nullptr;
	}
	int st;
	if (weighted) {
		st = pgq_csr_add_edges_weighted(entry.csr, edge_size, edge_size_count, rows, p_src, p_dst, p_eid, p_wi, p_wd);
	} else {
		st = pgq_csr_add_edges(entry.csr, edge_size, edge_size_count, rows, p_src, p_dst, p_eid);
	}
	if (st != PGQ_OK) {
		if (mirror) { // the host CSR is complete: remember the failure, path functions will upload it instead
			entry.error = pgq_last_error();
		} else {
			ThrowStatus(st);
		}
	}
	g_chunks++;
}

// ---- delete_csr -----------------------------------------------------------------------------------------------
static void DeleteCsrB200(const scalar_function_t &reference, DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CSRFunctionData>();
	GetB200State(info.context)->Drop(info.id);
	reference(args, state, result); // csr_list.erase(id), csr_deletion.cpp:10-20
}

// ---- reference functions that read the host CSR: materialise it first -----------------------------------------
static void HostConsumerB200(const scalar_function_t &reference, DataChunk &args, ExpressionState &state,
                             Vector &result) {
	auto &context = state.GetContext();
	auto pgq_state = context.registered_state->Get<DuckPGQState>("duckpgq");
	if (pgq_state) {
		GetB200State(context)->MaterialiseHost(*pgq_state);
	}
	reference(args, state, result);
}

template <int K>
struct TableWrap { // table functions are plain function pointers: one static slot per wrapped function
	static table_function_t function;
	static table_function_bind_t bind;
	static void Materialise(ClientContext &context) {
		auto pgq_state = context.registered_state->Get<DuckPGQState>("duckpgq");
		if (pgq_state) {
			GetB200State(context)->MaterialiseHost(*pgq_state);
		}
	}
	static unique_ptr<FunctionData> Bind(ClientContext &context, TableFunctionBindInput &input,
	                                     vector<LogicalType> &return_types, vector<string> &names) {
		Materialise(context);
		return bind(context, input, return_types, names);
	}
	static void Function(ClientContext &context, TableFunctionInput &data, DataChunk &output) {
		Materialise(context);
		function(context, data, output);
	}
};
template <int K>
table_function_t TableWrap<K>::function = nullptr;
template <int K>
table_function_bind_t TableWrap<K>::bind = nullptr;

// ---- iterativelength ----------------------------------------------------------------------------------
static void IterativeLengthB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);

	// the reference's three checks, iterativelength.cpp:41-51
	if (static_cast<idx_t>(info.csr_id) + 1 > duckpgq_state->csr_list.size()) {
		throw ConstraintException("Invalid ID");
	}
	auto csr_entry = duckpgq_state->csr_list.find(info.csr_id);
	if (csr_entry == duckpgq_state->csr_list.end()) {
		throw ConstraintException("Need to initialize CSR before doing shortest path");
	}
	if (!csr_entry->second->initialized_v) {
		throw ConstraintException("Need to initialize CSR before doing shortest path");
	}
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();

	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, *csr_entry->second, v_size);

	vector<int64_t> out_len(count);
	vector<uint8_t> out_valid(count);
	pgq_options opts = OptionsFromEnv();
	int st;
	// a chunk with enough rows for several lane batches is fanned out over the GPUs of PGQ_B200_DEVICES
	pgq_multi_csr *multi = count >= 512 ? GetB200State(info.context)->MultiFor(device_csr) : nullptr;
	if (multi) {
		st = pgq_multi_iterativelength(multi, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
		                               pairs.valid.data(), &opts, out_len.data(), out_valid.data(), nullptr);
	} else {
		st = pgq_iterativelength(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
		                         pairs.valid.data(), &opts, out_len.data(), out_valid.data(), nullptr);
	}
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_lengths++;
	g_pairs += static_cast<int64_t>(count);

	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<int64_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < count; i++) {
		result_data[i] = out_len[i]; // -1 under NULL, as iterativelength.cpp:100,138
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id); // iterativelength.cpp:142
}

// ---- iterativelengthbidirectional ----------------------------------------------------------------------
// iterativelength_bidirectional.cpp:43-153 on the device (pgq_iterativelength_bidirectional: the reference's 512-lane
// batches of the chunk's rows, one CSR, no fan-out -- a row's answer depends on the rows of its batch).  The reference
// reads its key columns through UnifiedVectorFormat::data, a byte pointer (l.61-62,104-110): row r searches from the
// BYTE at offset sel(r) of the column, and so does this callback.  Deviations in undefined territory (DESIGN §7): a
// NULL destination gives NULL, an id outside [0, v_size) fails, a missing CSR raises the texts of iterativelength.
static void IterativeLengthBidirectionalB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	if (static_cast<idx_t>(info.csr_id) + 1 > duckpgq_state->csr_list.size()) {
		throw ConstraintException("Invalid ID");
	}
	auto csr_entry = duckpgq_state->csr_list.find(info.csr_id);
	if (csr_entry == duckpgq_state->csr_list.end() || !csr_entry->second->initialized_v) {
		throw ConstraintException("Need to initialize CSR before doing shortest path");
	}
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, *csr_entry->second, v_size);
	UnifiedVectorFormat vsrc, vdst;
	args.data[2].ToUnifiedFormat(vsrc);
	args.data[3].ToUnifiedFormat(vdst);
	vector<int64_t> src(count), dst(count), out_len(count);
	vector<uint8_t> src_valid(count), dst_valid(count), out_valid(count);
	for (idx_t i = 0; i < count; i++) {
		auto sp = vsrc.sel->get_index(i), dp = vdst.sel->get_index(i);
		src_valid[i] = vsrc.validity.RowIsValid(sp) ? 1 : 0;
		dst_valid[i] = vdst.validity.RowIsValid(dp) ? 1 : 0;
		src[i] = vsrc.data[sp]; // (one byte, as the reference reads it)
		dst[i] = vdst.data[dp];
	}
	pgq_options opts = OptionsFromEnv();
	opts.lanes = 512;
	opts.flags = 0;
	int st = pgq_iterativelength_bidirectional(device_csr, static_cast<int64_t>(count), src.data(), dst.data(),
	                                           src_valid.data(), dst_valid.data(), &opts, out_len.data(),
	                                           out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_bidirectional++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<int64_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < count; i++) {
		result_data[i] = out_len[i]; // -1 under NULL, l.102-103,147
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id); // l.152
}

// ---- reachability ------------------------------------------------------------------------------------------------
// reachability.cpp:165-254 on the device (pgq_reachability: the rows of iterativelength by default, the reference's
// 512-lane batches with PGQ_B200_FLAGS=1).  Like the reference it reads both key columns through
// UnifiedVectorFormat::data, a byte pointer (l.177,181,26,242): row r searches from the BYTE at offset sel(r).  input_size
// is the v_size of the CSR; is_variant only picks the reference's traversal and is ignored.  Deviations in undefined
// territory (DESIGN §7): a NULL source or destination gives NULL, an id outside [0, input_size) fails, and NULL sources do
// not restart a batch.
static void ReachabilityB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	CSR *csr = duckpgq_state->GetCSR(info.csr_id); // "CSR not found with ID %d", l.192
	int64_t input_size = args.data[2].GetValue(0).GetValue<int64_t>();
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, *csr, input_size);
	UnifiedVectorFormat vsrc, vdst;
	args.data[3].ToUnifiedFormat(vsrc);
	args.data[4].ToUnifiedFormat(vdst);
	vector<int64_t> src(count), dst(count);
	vector<uint8_t> src_valid(count), dst_valid(count), out(count), out_valid(count);
	for (idx_t i = 0; i < count; i++) {
		auto sp = vsrc.sel->get_index(i), dp = vdst.sel->get_index(i);
		src_valid[i] = vsrc.validity.RowIsValid(sp) ? 1 : 0;
		dst_valid[i] = vdst.validity.RowIsValid(dp) ? 1 : 0;
		src[i] = vsrc.data[sp]; // (one byte, as the reference reads it)
		dst[i] = vdst.data[dp];
	}
	pgq_options opts = OptionsFromEnv();
	int st = pgq_reachability(device_csr, static_cast<int64_t>(count), src.data(), dst.data(), src_valid.data(),
	                          dst_valid.data(), &opts, out.data(), out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_reachability++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<bool>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < count; i++) {
		result_data[i] = out[i] != 0;
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id); // l.253
}

// ---- csr_get_w_type ------------------------------------------------------------------------------------
// csr_get_w_type.cpp:16-36 from the device build's weight type (0 unweighted -- also while no edge has arrived, as
// initialized_w == false --, 1 BIGINT, 2 DOUBLE): no host copy of the CSR.  A CSR without a usable device build is
// answered by the reference from the materialised host arrays.
static void CsrGetWTypeB200(const scalar_function_t &reference, DataChunk &args, ExpressionState &state,
                            Vector &result) {
	auto &info = state.expr.Cast<BoundFunctionExpression>().BindInfo()->Cast<CSRFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	duckpgq_state->GetCSR(info.id); // "CSR not found with ID %d", duckpgq_state.cpp:180-186
	auto entry = GetB200State(info.context)->Find(info.id);
	int wt = 0;
	if (!entry || !entry->error.empty() || pgq_csr_weight_type(entry->csr, &wt) != PGQ_OK) {
		HostConsumerB200(reference, args, state, result);
		return;
	}
	g_calls_w_type++;
	result.SetVectorType(VectorType::CONSTANT_VECTOR);
	ConstantVector::GetData<int32_t>(result)[0] = static_cast<int32_t>(wt);
}

// ---- shortestpath ---------------------------------------------------------------------------------------
static void ShortestPathB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);

	auto csr_entry = duckpgq_state->csr_list.find(info.csr_id); // shortest_path.cpp:49-57
	if (csr_entry == duckpgq_state->csr_list.end()) {
		throw ConstraintException("Invalid ID");
	}
	if (!csr_entry->second->initialized_v) {
		throw ConstraintException("Need to initialize CSR before doing shortest path");
	}
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();

	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, *csr_entry->second, v_size);

	vector<int64_t> offsets(count), lengths(count);
	vector<uint8_t> out_valid(count);
	int64_t *elems = nullptr;
	int64_t total = 0;
	pgq_options opts = OptionsFromEnv();
	int st = pgq_shortestpath(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                          pairs.valid.data(), &opts, offsets.data(), lengths.data(), out_valid.data(), &elems,
	                          &total, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_paths++;
	g_pairs += static_cast<int64_t>(count);

	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<list_entry_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	ListVector::Reserve(result, static_cast<idx_t>(total));
	if (total > 0) {
		auto child_data = FlatVector::GetDataMutable<int64_t>(ListVector::GetChildMutable(result));
		memcpy(child_data, elems, static_cast<size_t>(total) * sizeof(int64_t));
	}
	ListVector::SetListSize(result, static_cast<idx_t>(total));
	pgq_free(elems);
	for (idx_t i = 0; i < count; i++) {
		result_data[i].offset = static_cast<idx_t>(offsets[i]);
		result_data[i].length = static_cast<idx_t>(lengths[i]);
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id); // shortest_path.cpp:206
}

// ---- shortest_path_count / all_shortest_paths (no reference function) ----------------------------------------
// Every shortest path of a row (include/duckpgq_b200.h, pgq_shortest_path_count / pgq_all_shortest_paths), called as
// raw UDFs over the CSR CTE: the MATCH rewriter stays the reference's, which rejects ALL SHORTEST.  The binds are
// shortestpath's (IterativeLengthBind: constant id, the mark for deletion); all_shortest_paths' also wants a constant
// max_paths >= 0 (0 = every path).  The CSR lookups are shortestpath's (shortest_path.cpp:49-57).
static CSR &ShortestPathCsr(DuckPGQState &duckpgq_state, int32_t csr_id) {
	auto csr_entry = duckpgq_state.csr_list.find(csr_id);
	if (csr_entry == duckpgq_state.csr_list.end()) {
		throw ConstraintException("Invalid ID");
	}
	if (!csr_entry->second->initialized_v) {
		throw ConstraintException("Need to initialize CSR before doing shortest path");
	}
	return *csr_entry->second;
}

static void ShortestPathCountB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	CSR &csr = ShortestPathCsr(*duckpgq_state, info.csr_id);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, csr, v_size);
	vector<int64_t> out_count(count);
	vector<uint8_t> out_valid(count);
	pgq_options opts = OptionsFromEnv();
	int st = pgq_shortest_path_count(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                                 pairs.valid.data(), nullptr, &opts, out_count.data(), out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_path_count++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<int64_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < count; i++) {
		result_data[i] = out_count[i];
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id);
}

static unique_ptr<FunctionData> AllShortestPathsBind(BindScalarFunctionInput &input) {
	auto &arguments = input.GetArguments();
	if (!arguments[4]->IsFoldable()) {
		throw InvalidInputException("max_paths must be constant.");
	}
	auto max_paths = ExpressionExecutor::EvaluateScalar(input.GetClientContext(), *arguments[4]);
	if (max_paths.IsNull() || max_paths.GetValue<int64_t>() < 0) {
		throw InvalidInputException("max_paths must be 0 (every path) or more.");
	}
	return IterativeLengthFunctionData::IterativeLengthBind(input);
}

static void AllShortestPathsB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	CSR &csr = ShortestPathCsr(*duckpgq_state, info.csr_id);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	int64_t max_paths = args.data[4].GetValue(0).GetValue<int64_t>(); // (constant: AllShortestPathsBind)
	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, csr, v_size);
	vector<int64_t> out_count(count), npaths(count), path_len(count), offsets(count);
	vector<uint8_t> out_valid(count);
	int64_t *elems = nullptr;
	int64_t total = 0;
	pgq_options opts = OptionsFromEnv();
	int st = pgq_all_shortest_paths(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                                pairs.valid.data(), nullptr, &opts, max_paths, out_count.data(), npaths.data(),
	                                path_len.data(), offsets.data(), out_valid.data(), &elems, &total, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_all_shortest++;
	g_pairs += static_cast<int64_t>(count);
	idx_t lists = 0;
	for (idx_t i = 0; i < count; i++) {
		lists += static_cast<idx_t>(npaths[i]);
	}
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<list_entry_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	ListVector::Reserve(result, lists);
	auto &inner = ListVector::GetChildMutable(result);
	ListVector::Reserve(inner, static_cast<idx_t>(total));
	if (total > 0) {
		auto leaf = FlatVector::GetDataMutable<int64_t>(ListVector::GetChildMutable(inner));
		memcpy(leaf, elems, static_cast<size_t>(total) * sizeof(int64_t));
	}
	ListVector::SetListSize(inner, static_cast<idx_t>(total));
	pgq_free(elems);
	auto inner_data = FlatVector::GetDataMutable<list_entry_t>(inner);
	idx_t li = 0;
	for (idx_t i = 0; i < count; i++) {
		result_data[i].offset = li;
		result_data[i].length = static_cast<idx_t>(npaths[i]);
		for (int64_t k = 0; k < npaths[i]; k++, li++) {
			inner_data[li].offset = static_cast<idx_t>(offsets[i] + k * path_len[i]);
			inner_data[li].length = static_cast<idx_t>(path_len[i]);
		}
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	ListVector::SetListSize(result, lists);
	duckpgq_state->csr_to_delete.insert(info.csr_id);
}

// ---- shortest_k_paths (no reference function) ---------------------------------------------------------------
// The k shortest walks of a row (include/duckpgq_b200.h, pgq_shortest_k_paths), called as a raw UDF over the CSR CTE:
// the MATCH rewriter stays the reference's, which rejects SHORTEST k (match.cpp:84-86).  The bind is shortestpath's
// and also wants a constant k >= 1; the CSR lookup is shortestpath's.
static void CheckConstantK(BindScalarFunctionInput &input) {
	auto &arguments = input.GetArguments();
	if (!arguments[4]->IsFoldable()) {
		throw InvalidInputException("k must be constant.");
	}
	auto k = ExpressionExecutor::EvaluateScalar(input.GetClientContext(), *arguments[4]);
	if (k.IsNull() || k.GetValue<int64_t>() < 1) {
		throw InvalidInputException("k must be 1 or more.");
	}
}

static unique_ptr<FunctionData> ShortestKPathsBind(BindScalarFunctionInput &input) {
	CheckConstantK(input);
	return IterativeLengthFunctionData::IterativeLengthBind(input);
}

// SQL/PGQ's path mode by name, any case (PGQPathMode's WALK, TRAIL, ACYCLIC, SIMPLE), or -1
static int32_t PathModeId(const string &name) {
	const string up = StringUtil::Upper(name);
	return up == "WALK" ? PGQ_PATH_WALK
	       : up == "TRAIL" ? PGQ_PATH_TRAIL
	       : up == "ACYCLIC" ? PGQ_PATH_ACYCLIC
	       : up == "SIMPLE" ? PGQ_PATH_SIMPLE
	                        : -1;
}

// shortest_k_paths(INTEGER, BIGINT, BIGINT, BIGINT, BIGINT k, VARCHAR mode): the 5-argument bind, and a constant mode
// that names a path mode
static void CheckConstantMode(BindScalarFunctionInput &input) {
	auto &arguments = input.GetArguments();
	if (!arguments[5]->IsFoldable()) {
		throw InvalidInputException("the path mode must be constant.");
	}
	auto mode = ExpressionExecutor::EvaluateScalar(input.GetClientContext(), *arguments[5]);
	if (mode.IsNull() || PathModeId(mode.GetValue<string>()) < 0) {
		throw InvalidInputException("the path mode must be WALK, TRAIL, ACYCLIC or SIMPLE.");
	}
}

static unique_ptr<FunctionData> ShortestKPathsModeBind(BindScalarFunctionInput &input) {
	CheckConstantMode(input);
	return ShortestKPathsBind(input);
}

// The rows' path lists of pgq_shortest_k_paths_mode / pgq_shortest_k_groups as LIST(LIST(BIGINT)): row i holds paths
// first[i] .. first[i] + npaths[i] - 1, path j is elems[offsets[j] .. offsets[j + 1]), and a row with valid[i] = 0 is
// NULL.  The caller frees offsets and elems.
static void SetPathLists(Vector &result, idx_t count, const int64_t *offsets, const int64_t *elems, int64_t paths,
                         const vector<int64_t> &first, const vector<int64_t> &npaths, const vector<uint8_t> &valid) {
	const idx_t total = static_cast<idx_t>(offsets[paths]);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<list_entry_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	ListVector::Reserve(result, static_cast<idx_t>(paths));
	auto &inner = ListVector::GetChildMutable(result);
	ListVector::Reserve(inner, total);
	if (total > 0) {
		auto leaf = FlatVector::GetDataMutable<int64_t>(ListVector::GetChildMutable(inner));
		memcpy(leaf, elems, total * sizeof(int64_t));
	}
	ListVector::SetListSize(inner, total);
	auto inner_data = FlatVector::GetDataMutable<list_entry_t>(inner);
	for (int64_t j = 0; j < paths; j++) {
		inner_data[j].offset = static_cast<idx_t>(offsets[j]);
		inner_data[j].length = static_cast<idx_t>(offsets[j + 1] - offsets[j]);
	}
	for (idx_t i = 0; i < count; i++) {
		result_data[i].offset = static_cast<idx_t>(first[i]);
		result_data[i].length = static_cast<idx_t>(npaths[i]);
		if (!valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	ListVector::SetListSize(result, static_cast<idx_t>(paths));
}

// Both overloads: the rows' lists of pgq_shortest_k_paths_mode (WALK is pgq_shortest_k_paths itself)
static void ShortestKPathsRows(DataChunk &args, ExpressionState &state, Vector &result, int32_t mode) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	CSR &csr = ShortestPathCsr(*duckpgq_state, info.csr_id);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	int64_t k = args.data[4].GetValue(0).GetValue<int64_t>(); // (constant: ShortestKPathsBind)
	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, csr, v_size);
	vector<int64_t> npaths(count), first(count);
	vector<uint8_t> out_valid(count);
	int64_t *offsets = nullptr, *elems = nullptr;
	int64_t walks = 0;
	pgq_options opts = OptionsFromEnv();
	int st = pgq_shortest_k_paths_mode(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                                   pairs.valid.data(), nullptr, &opts, k, mode, npaths.data(), first.data(),
	                                   out_valid.data(), &offsets, &elems, &walks, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_pairs += static_cast<int64_t>(count);
	SetPathLists(result, count, offsets, elems, walks, first, npaths, out_valid);
	pgq_free(offsets);
	pgq_free(elems);
	duckpgq_state->csr_to_delete.insert(info.csr_id);
}

static void ShortestKPathsB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	ShortestKPathsRows(args, state, result, PGQ_PATH_WALK);
	g_calls_shortest_k++;
}

static void ShortestKPathsModeB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	// (constant and valid: ShortestKPathsModeBind)
	ShortestKPathsRows(args, state, result, PathModeId(args.data[5].GetValue(0).GetValue<string>()));
	g_calls_shortest_k_mode++;
}

// ---- shortest_k_groups (no reference function) --------------------------------------------------------------
// Every path of the k shortest lengths of a row (include/duckpgq_b200.h, pgq_shortest_k_groups), SQL/PGQ's SHORTEST k
// GROUP, called as a raw UDF over the CSR CTE like shortest_k_paths.
// shortest_k_groups(INTEGER, BIGINT, BIGINT, BIGINT, BIGINT k, BIGINT max_paths[, VARCHAR mode]): shortest_k_paths'
// checks of k and the mode, and a constant max_paths >= 0
static unique_ptr<FunctionData> ShortestKGroupsBind(BindScalarFunctionInput &input) {
	auto &arguments = input.GetArguments();
	if (!arguments[5]->IsFoldable()) {
		throw InvalidInputException("max_paths must be constant.");
	}
	auto max_paths = ExpressionExecutor::EvaluateScalar(input.GetClientContext(), *arguments[5]);
	if (max_paths.IsNull() || max_paths.GetValue<int64_t>() < 0) {
		throw InvalidInputException("max_paths must be 0 (every path) or more.");
	}
	if (arguments.size() > 6) {
		if (!arguments[6]->IsFoldable()) {
			throw InvalidInputException("the path mode must be constant.");
		}
		auto mode = ExpressionExecutor::EvaluateScalar(input.GetClientContext(), *arguments[6]);
		if (mode.IsNull() || PathModeId(mode.GetValue<string>()) < 0) {
			throw InvalidInputException("the path mode must be WALK, TRAIL, ACYCLIC or SIMPLE.");
		}
	}
	return ShortestKPathsBind(input);
}

static void ShortestKGroupsB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	CSR &csr = ShortestPathCsr(*duckpgq_state, info.csr_id);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	// (constant and valid: ShortestKGroupsBind)
	int64_t k = args.data[4].GetValue(0).GetValue<int64_t>();
	int64_t max_paths = args.data[5].GetValue(0).GetValue<int64_t>();
	int32_t mode = args.ColumnCount() > 6 ? PathModeId(args.data[6].GetValue(0).GetValue<string>()) : PGQ_PATH_WALK;
	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, csr, v_size);
	vector<int64_t> ngroups(count), last_len(count), npaths(count), first(count);
	vector<uint8_t> complete(count), out_valid(count);
	int64_t *offsets = nullptr, *elems = nullptr;
	int64_t paths = 0;
	pgq_options opts = OptionsFromEnv();
	int st = pgq_shortest_k_groups(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                               pairs.valid.data(), nullptr, &opts, k, mode, max_paths, nullptr, ngroups.data(),
	                               last_len.data(), complete.data(), npaths.data(), first.data(), out_valid.data(),
	                               &offsets, &elems, &paths, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_shortest_k_groups++;
	g_pairs += static_cast<int64_t>(count);
	SetPathLists(result, count, offsets, elems, paths, first, npaths, out_valid);
	pgq_free(offsets);
	pgq_free(elems);
	duckpgq_state->csr_to_delete.insert(info.csr_id);
}

// shortest_k_groups_count(INTEGER, BIGINT, BIGINT, BIGINT, BIGINT k) -> BIGINT: WALK's N, saturated at INT64_MAX, NULL
// for a row without a walk
static void ShortestKGroupsCountB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<IterativeLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	CSR &csr = ShortestPathCsr(*duckpgq_state, info.csr_id);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	int64_t k = args.data[4].GetValue(0).GetValue<int64_t>(); // (constant: ShortestKPathsBind)
	PairColumns pairs(args);
	idx_t count = args.size();
	auto device_csr = GetB200State(info.context)->ForPathFunction(info.csr_id, csr, v_size);
	vector<int64_t> out_count(count), ngroups(count), last_len(count);
	vector<uint8_t> out_valid(count);
	pgq_options opts = OptionsFromEnv();
	int st = pgq_shortest_k_groups_count(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                                     pairs.valid.data(), nullptr, &opts, k, out_count.data(), ngroups.data(),
	                                     last_len.data(), out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_shortest_k_groups_count++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<int64_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < count; i++) {
		result_data[i] = out_count[i];
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id);
}

// ---- cheapest_path_length -------------------------------------------------------------------------------
// cheapest_path_length.cpp:138-160: batched Bellman-Ford over the weighted CSR, BIGINT or DOUBLE result as
// the bind decided (cheapest_path_length_function_data.cpp:26-30).  The bind stays the reference's.
static void CheapestPathLengthB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CheapestPathLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	int64_t v_size = args.data[1].GetValue(0).GetValue<int64_t>();
	CSR *host = duckpgq_state->GetCSR(info.csr_id); // "CSR not found with ID", duckpgq_state.cpp:180-186
	auto b200 = GetB200State(info.context);
	auto entry = b200->Find(info.csr_id);
	int wt = 0;
	if (!entry || !entry->error.empty() || pgq_csr_finalize(entry->csr) != PGQ_OK ||
	    pgq_csr_weight_type(entry->csr, &wt) != PGQ_OK || wt == 0) {
		throw InvalidInputException("duckpgq_b200: cheapest_path_length needs a weighted CSR built through create_csr_edge");
	}
	(void)host;
	idx_t count = args.size();
	UnifiedVectorFormat vsrc, vdst;
	args.data[2].ToUnifiedFormat(vsrc);
	args.data[3].ToUnifiedFormat(vdst);
	auto src_data = reinterpret_cast<const int64_t *>(vsrc.data);
	auto dst_data = reinterpret_cast<const int64_t *>(vdst.data);
	vector<int64_t> src(count), dst(count);
	vector<uint8_t> src_valid(count), dst_valid(count), out_valid(count);
	for (idx_t i = 0; i < count; i++) {
		auto sp = vsrc.sel->get_index(i), dp = vdst.sel->get_index(i);
		src_valid[i] = vsrc.validity.RowIsValid(sp);
		dst_valid[i] = vdst.validity.RowIsValid(dp);
		src[i] = src_valid[i] ? src_data[sp] : 0;
		dst[i] = dst_valid[i] ? dst_data[dp] : 0;
	}
	vector<int64_t> out(count); // raw 8-byte costs: int64 or double as the CSR's weights
	int st = pgq_cheapest_path_length(entry->csr, static_cast<int64_t>(count), src.data(), dst.data(), src_valid.data(),
	                                  dst_valid.data(), out.data(), out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_cheapest++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto &result_validity = FlatVector::ValidityMutable(result);
	memcpy(FlatVector::GetDataMutable<int64_t>(result), out.data(), count * sizeof(int64_t)); // (BIGINT and DOUBLE are both 8 bytes)
	for (idx_t i = 0; i < count; i++) {
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id); // cheapest_path_length.cpp:160
}

// ---- cheapest_path (no reference function) ----------------------------------------------------------------
// The cheapest path itself as shortestpath's list (include/duckpgq_b200.h, pgq_cheapest_path).  The bind does what
// CheapestPathLengthBind does (cheapest_path_length_function_data.cpp:7-31: constant id, GetCSR, the mark for
// deletion, the weights check), then returns LIST(BIGINT) whatever the weight type.
static unique_ptr<FunctionData> CheapestPathBind(BindScalarFunctionInput &input) {
	auto &context = input.GetClientContext();
	auto &arguments = input.GetArguments();
	if (!arguments[0]->IsFoldable()) {
		throw InvalidInputException("Id must be constant.");
	}
	auto duckpgq_state = GetDuckPGQState(context);
	int32_t csr_id = ExpressionExecutor::EvaluateScalar(context, *arguments[0]).GetValue<int32_t>();
	CSR *csr = duckpgq_state->GetCSR(csr_id);
	duckpgq_state->csr_to_delete.insert(csr_id);
	if (!(csr->initialized_v && csr->initialized_e && csr->initialized_w)) {
		throw ConstraintException("Need to initialize CSR before doing cheapest path");
	}
	input.GetBoundFunction().SetReturnType(LogicalType::LIST(LogicalType::BIGINT));
	return make_uniq<CheapestPathLengthFunctionData>(context, csr_id);
}

static void CheapestPathB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CheapestPathLengthFunctionData>();
	auto duckpgq_state = GetDuckPGQState(info.context);
	(void)duckpgq_state->GetCSR(info.csr_id); // "CSR not found with ID", duckpgq_state.cpp:180-186
	auto entry = GetB200State(info.context)->Find(info.csr_id);
	int wt = 0;
	if (!entry || !entry->error.empty() || pgq_csr_finalize(entry->csr) != PGQ_OK ||
	    pgq_csr_weight_type(entry->csr, &wt) != PGQ_OK || wt == 0) {
		throw InvalidInputException("duckpgq_b200: cheapest_path needs a weighted CSR built through create_csr_edge");
	}
	idx_t count = args.size();
	UnifiedVectorFormat vsrc, vdst;
	args.data[2].ToUnifiedFormat(vsrc);
	args.data[3].ToUnifiedFormat(vdst);
	auto src_data = reinterpret_cast<const int64_t *>(vsrc.data);
	auto dst_data = reinterpret_cast<const int64_t *>(vdst.data);
	vector<int64_t> src(count), dst(count), offsets(count), lengths(count);
	vector<uint8_t> src_valid(count), dst_valid(count), out_valid(count);
	for (idx_t i = 0; i < count; i++) {
		auto sp = vsrc.sel->get_index(i), dp = vdst.sel->get_index(i);
		src_valid[i] = vsrc.validity.RowIsValid(sp);
		dst_valid[i] = vdst.validity.RowIsValid(dp);
		src[i] = src_valid[i] ? src_data[sp] : 0;
		dst[i] = dst_valid[i] ? dst_data[dp] : 0;
	}
	int64_t *elems = nullptr;
	int64_t total = 0;
	int st = pgq_cheapest_path(entry->csr, static_cast<int64_t>(count), src.data(), dst.data(), src_valid.data(),
	                           dst_valid.data(), offsets.data(), lengths.data(), out_valid.data(), &elems, &total, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_cheapest_path++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<list_entry_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	ListVector::Reserve(result, static_cast<idx_t>(total));
	if (total > 0) {
		auto child_data = FlatVector::GetDataMutable<int64_t>(ListVector::GetChildMutable(result));
		memcpy(child_data, elems, static_cast<size_t>(total) * sizeof(int64_t));
	}
	ListVector::SetListSize(result, static_cast<idx_t>(total));
	pgq_free(elems);
	for (idx_t i = 0; i < count; i++) {
		result_data[i].offset = static_cast<idx_t>(offsets[i]);
		result_data[i].length = static_cast<idx_t>(lengths[i]);
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	duckpgq_state->csr_to_delete.insert(info.csr_id);
}

// ---- cheapest_path_count / all_cheapest_paths (no reference function) ------------------------------------------
// Every cheapest path of a row (include/duckpgq_b200.h, pgq_cheapest_path_count / pgq_all_cheapest_paths).  The binds
// are cheapest_path's (constant id, GetCSR, the mark for deletion, the weights check) with their own result types;
// all_cheapest_paths' max_paths is a constant >= 0.
static unique_ptr<FunctionData> CheapestPathCountBind(BindScalarFunctionInput &input) {
	auto data = CheapestPathBind(input);
	input.GetBoundFunction().SetReturnType(LogicalType::BIGINT);
	return data;
}

static unique_ptr<FunctionData> AllCheapestPathsBind(BindScalarFunctionInput &input) {
	auto &arguments = input.GetArguments();
	if (!arguments[4]->IsFoldable()) {
		throw InvalidInputException("max_paths must be constant.");
	}
	auto max_paths = ExpressionExecutor::EvaluateScalar(input.GetClientContext(), *arguments[4]);
	if (max_paths.IsNull() || max_paths.GetValue<int64_t>() < 0) {
		throw InvalidInputException("max_paths must be 0 (every path) or more.");
	}
	auto data = CheapestPathBind(input);
	input.GetBoundFunction().SetReturnType(LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)));
	return data;
}

// The weighted device CSR of a cheapest-path call and its rows' ids and validity (cheapest_path's lookup)
static pgq_csr *CheapestCsr(ClientContext &context, int32_t csr_id, const char *what) {
	auto duckpgq_state = GetDuckPGQState(context);
	(void)duckpgq_state->GetCSR(csr_id); // "CSR not found with ID", duckpgq_state.cpp:180-186
	auto entry = GetB200State(context)->Find(csr_id);
	int wt = 0;
	if (!entry || !entry->error.empty() || pgq_csr_finalize(entry->csr) != PGQ_OK ||
	    pgq_csr_weight_type(entry->csr, &wt) != PGQ_OK || wt == 0) {
		throw InvalidInputException("duckpgq_b200: %s needs a weighted CSR built through create_csr_edge", what);
	}
	return entry->csr;
}

struct CheapestPairs {
	vector<int64_t> src, dst;
	vector<uint8_t> src_valid, dst_valid;
	explicit CheapestPairs(DataChunk &args) {
		idx_t count = args.size();
		UnifiedVectorFormat vsrc, vdst;
		args.data[2].ToUnifiedFormat(vsrc);
		args.data[3].ToUnifiedFormat(vdst);
		auto src_data = reinterpret_cast<const int64_t *>(vsrc.data);
		auto dst_data = reinterpret_cast<const int64_t *>(vdst.data);
		src.resize(count);
		dst.resize(count);
		src_valid.resize(count);
		dst_valid.resize(count);
		for (idx_t i = 0; i < count; i++) {
			auto sp = vsrc.sel->get_index(i), dp = vdst.sel->get_index(i);
			src_valid[i] = vsrc.validity.RowIsValid(sp);
			dst_valid[i] = vdst.validity.RowIsValid(dp);
			src[i] = src_valid[i] ? src_data[sp] : 0;
			dst[i] = dst_valid[i] ? dst_data[dp] : 0;
		}
	}
};

static void CheapestPathCountB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CheapestPathLengthFunctionData>();
	pgq_csr *device_csr = CheapestCsr(info.context, info.csr_id, "cheapest_path_count");
	idx_t count = args.size();
	CheapestPairs pairs(args);
	vector<int64_t> out_count(count);
	vector<uint8_t> out_valid(count);
	int st = pgq_cheapest_path_count(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                                 pairs.src_valid.data(), pairs.dst_valid.data(), out_count.data(), out_valid.data(),
	                                 nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_cheapest_count++;
	g_pairs += static_cast<int64_t>(count);
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<int64_t>(result);
	ValidityMask &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < count; i++) {
		result_data[i] = out_count[i];
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
	GetDuckPGQState(info.context)->csr_to_delete.insert(info.csr_id);
}

static void AllCheapestPathsB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CheapestPathLengthFunctionData>();
	pgq_csr *device_csr = CheapestCsr(info.context, info.csr_id, "all_cheapest_paths");
	int64_t max_paths = args.data[4].GetValue(0).GetValue<int64_t>(); // (constant: AllCheapestPathsBind)
	idx_t count = args.size();
	CheapestPairs pairs(args);
	vector<int64_t> out_count(count), npaths(count), first(count);
	vector<uint8_t> out_valid(count);
	int64_t *offsets = nullptr, *elems = nullptr;
	int64_t paths = 0;
	int st = pgq_all_cheapest_paths(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                                pairs.src_valid.data(), pairs.dst_valid.data(), max_paths, out_count.data(),
	                                npaths.data(), first.data(), out_valid.data(), &offsets, &elems, &paths, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_all_cheapest++;
	g_pairs += static_cast<int64_t>(count);
	SetPathLists(result, count, offsets, elems, paths, first, npaths, out_valid);
	pgq_free(offsets);
	pgq_free(elems);
	GetDuckPGQState(info.context)->csr_to_delete.insert(info.csr_id);
}

// ---- cheapest_k_paths / cheapest_k_costs (no reference function) ----------------------------------------------
// The k cheapest paths of a row in a path mode and their costs (include/duckpgq_b200.h, pgq_cheapest_k_paths),
// SQL/PGQ's CHEAPEST k, raw UDFs over the weighted CSR CTE like cheapest_path.  The binds are cheapest_path's with
// shortest_k_paths' checks of a constant k >= 1 and, with a 6th argument, of a constant path mode.  cheapest_k_costs
// returns a LIST of the CSR's weight type, chosen as cheapest_path_length's bind chooses its result
// (cheapest_path_length_function_data.cpp:25-29).  Both count as cheapest_k_paths_calls.
static unique_ptr<FunctionData> CheapestKBind(BindScalarFunctionInput &input) {
	CheckConstantK(input);
	if (input.GetArguments().size() > 5) {
		CheckConstantMode(input);
	}
	return CheapestPathBind(input);
}

static unique_ptr<FunctionData> CheapestKPathsBind(BindScalarFunctionInput &input) {
	auto data = CheapestKBind(input);
	input.GetBoundFunction().SetReturnType(LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)));
	return data;
}

static unique_ptr<FunctionData> CheapestKCostsBind(BindScalarFunctionInput &input) {
	auto data = CheapestKBind(input);
	CSR *csr = GetDuckPGQState(input.GetClientContext())->GetCSR(data->Cast<CheapestPathLengthFunctionData>().csr_id);
	input.GetBoundFunction().SetReturnType(LogicalType::LIST(csr->w.empty() ? LogicalType::DOUBLE : LogicalType::BIGINT));
	return data;
}

// Both UDFs: pgq_cheapest_k_paths over the chunk's rows, then the rows' path lists, or their cost lists (the raw 8-byte
// costs: BIGINT and DOUBLE have the same width).  opts stay null: the call picks its own lane width.
static void CheapestKRows(DataChunk &args, ExpressionState &state, Vector &result, bool costs) {
	auto &func_expr = state.expr.Cast<BoundFunctionExpression>();
	auto &info = func_expr.BindInfo()->Cast<CheapestPathLengthFunctionData>();
	pgq_csr *device_csr = CheapestCsr(info.context, info.csr_id, costs ? "cheapest_k_costs" : "cheapest_k_paths");
	int64_t k = args.data[4].GetValue(0).GetValue<int64_t>(); // (constant: CheapestKBind)
	int32_t mode = args.ColumnCount() > 5 ? PathModeId(args.data[5].GetValue(0).GetValue<string>()) : PGQ_PATH_WALK;
	idx_t count = args.size();
	CheapestPairs pairs(args);
	vector<int64_t> npaths(count), first(count);
	vector<uint8_t> out_valid(count);
	int64_t *offsets = nullptr, *elems = nullptr;
	void *cost_bits = nullptr;
	int64_t paths = 0;
	int st = pgq_cheapest_k_paths(device_csr, static_cast<int64_t>(count), pairs.src.data(), pairs.dst.data(),
	                              pairs.src_valid.data(), pairs.dst_valid.data(), nullptr, k, mode, npaths.data(),
	                              first.data(), out_valid.data(), &offsets, &elems, costs ? &cost_bits : nullptr, &paths,
	                              nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_cheapest_k++;
	g_pairs += static_cast<int64_t>(count);
	if (!costs) {
		SetPathLists(result, count, offsets, elems, paths, first, npaths, out_valid);
	} else {
		result.SetVectorType(VectorType::FLAT_VECTOR);
		auto result_data = FlatVector::GetDataMutable<list_entry_t>(result);
		ValidityMask &result_validity = FlatVector::ValidityMutable(result);
		ListVector::Reserve(result, static_cast<idx_t>(paths));
		if (paths > 0) {
			memcpy(FlatVector::GetDataMutable<int64_t>(ListVector::GetChildMutable(result)), cost_bits,
			       static_cast<size_t>(paths) * sizeof(int64_t));
		}
		ListVector::SetListSize(result, static_cast<idx_t>(paths));
		for (idx_t i = 0; i < count; i++) {
			result_data[i].offset = static_cast<idx_t>(first[i]);
			result_data[i].length = static_cast<idx_t>(npaths[i]);
			if (!out_valid[i]) {
				result_validity.SetInvalid(i);
			}
		}
	}
	pgq_free(offsets);
	pgq_free(elems);
	pgq_free(cost_bits);
	GetDuckPGQState(info.context)->csr_to_delete.insert(info.csr_id);
}

static void CheapestKPathsB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	CheapestKRows(args, state, result, false);
}

static void CheapestKCostsB200Function(DataChunk &args, ExpressionState &state, Vector &result) {
	CheapestKRows(args, state, result, true);
}

// ---- local_clustering_coefficient / pagerank / weakly_connected_component ---------------------------------------
// Registered through WrapScalar, so the signatures and binds are the reference's; the reference callback is not
// called.  The device CSR is found like a path function's (the device build, or an upload of the host CSR).
static pgq_csr *ForAnalytics(ClientContext &context, int32_t csr_id, const char *not_initialized) {
	auto duckpgq_state = GetDuckPGQState(context);
	auto csr_entry = duckpgq_state->csr_list.find(csr_id); // e.g. pagerank.cpp:17-24
	if (csr_entry == duckpgq_state->csr_list.end()) {
		throw ConstraintException("CSR not found. Is the graph populated?");
	}
	CSR &host = *csr_entry->second;
	auto b200 = GetB200State(context);
	auto entry = b200->Find(csr_id);
	// initialized_e: in mode `skip` the host arrays stay empty, and edges that reached the device build count
	const bool edges = host.initialized_e || (entry && entry->edges_started);
	if (!(host.initialized_v && edges)) {
		throw ConstraintException(not_initialized);
	}
	return b200->ForPathFunction(csr_id, host, static_cast<int64_t>(host.vsize) - 2);
}

// The source column (args.data[1]) as contiguous ids + validity.
struct SourceColumn {
	vector<int64_t> src;
	vector<uint8_t> valid;
	SourceColumn(DataChunk &args) {
		Column<int64_t> col(args.data[1], args.size());
		src.assign(col.data, col.data + args.size());
		valid.resize(args.size());
		for (idx_t i = 0; i < args.size(); i++) {
			valid[i] = col.RowIsValid(i) ? 1 : 0;
		}
	}
};

template <class T>
static void WriteAnalyticsResult(Vector &result, const vector<T> &out, const vector<uint8_t> &out_valid) {
	result.SetVectorType(VectorType::FLAT_VECTOR);
	auto result_data = FlatVector::GetDataMutable<T>(result);
	auto &result_validity = FlatVector::ValidityMutable(result);
	for (idx_t i = 0; i < out.size(); i++) {
		result_data[i] = out[i];
		if (!out_valid[i]) {
			result_validity.SetInvalid(i);
		}
	}
}

static void LocalClusteringCoefficientB200(const scalar_function_t &, DataChunk &args, ExpressionState &state,
                                           Vector &result) {
	auto &info = state.expr.Cast<BoundFunctionExpression>().BindInfo()->Cast<LocalClusteringCoefficientFunctionData>();
	pgq_csr *csr = ForAnalytics(info.context, info.csr_id,
	                            "Need to initialize CSR before doing local clustering coefficient.");
	SourceColumn src(args);
	vector<float> out(args.size());
	vector<uint8_t> out_valid(args.size());
	int st = pgq_local_clustering_coefficient(csr, static_cast<int64_t>(args.size()), src.src.data(), src.valid.data(),
	                                          out.data(), out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_lcc++;
	WriteAnalyticsResult(result, out, out_valid);
	GetDuckPGQState(info.context)->csr_to_delete.insert(info.csr_id); // local_clustering_coefficient.cpp:71
}

static void PageRankB200(const scalar_function_t &, DataChunk &args, ExpressionState &state, Vector &result) {
	auto &info = state.expr.Cast<BoundFunctionExpression>().BindInfo()->Cast<PageRankFunctionData>();
	pgq_csr *csr = ForAnalytics(info.context, info.csr_id, "Need to initialize CSR before running PageRank.");
	SourceColumn src(args);
	vector<double> out(args.size());
	vector<uint8_t> out_valid(args.size());
	int st = pgq_pagerank(csr, static_cast<int64_t>(args.size()), src.src.data(), src.valid.data(), out.data(),
	                      out_valid.data(), nullptr, nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_pagerank++;
	WriteAnalyticsResult(result, out, out_valid);
	GetDuckPGQState(info.context)->csr_to_delete.insert(info.csr_id); // pagerank.cpp:110
}

static void WeaklyConnectedComponentB200(const scalar_function_t &, DataChunk &args, ExpressionState &state,
                                         Vector &result) {
	auto &info = state.expr.Cast<BoundFunctionExpression>().BindInfo()->Cast<WeaklyConnectedComponentFunctionData>();
	pgq_csr *csr = ForAnalytics(info.context, info.csr_id,
	                            "Need to initialize CSR before doing weakly connected components.");
	SourceColumn src(args);
	vector<int64_t> out(args.size());
	vector<uint8_t> out_valid(args.size());
	int st = pgq_weakly_connected_component(csr, static_cast<int64_t>(args.size()), src.src.data(), src.valid.data(),
	                                        out.data(), out_valid.data(), nullptr);
	if (st != PGQ_OK) {
		ThrowStatus(st);
	}
	g_calls_wcc++;
	WriteAnalyticsResult(result, out, out_valid);
	GetDuckPGQState(info.context)->csr_to_delete.insert(info.csr_id); // weakly_connected_component.cpp:103
}

// ---- introspection: proves which implementation served the query ------------------------------------------
// duckpgq_b200_stats() -> 'iterativelength_calls=..,shortestpath_calls=..,pairs=..,csr_uploads=..,...'
static void B200StatsFunction(DataChunk &args, ExpressionState &state, Vector &result) {
	string text = "iterativelength_calls=" + std::to_string(g_calls_lengths.load()) +
	              ",shortestpath_calls=" + std::to_string(g_calls_paths.load()) +
	              ",cheapest_path_length_calls=" + std::to_string(g_calls_cheapest.load()) +
	              ",pairs=" + std::to_string(g_pairs.load()) + ",csr_uploads=" + std::to_string(g_uploads.load()) +
	              ",csr_device_builds=" + std::to_string(g_device_builds.load()) +
	              ",csr_chunks=" + std::to_string(g_chunks.load()) +
	              ",host_csr_materialisations=" + std::to_string(g_materialized.load()) +
	              ",local_clustering_coefficient_calls=" + std::to_string(g_calls_lcc.load()) +
	              ",pagerank_calls=" + std::to_string(g_calls_pagerank.load()) +
	              ",weakly_connected_component_calls=" + std::to_string(g_calls_wcc.load()) +
	              ",iterativelengthbidirectional_calls=" + std::to_string(g_calls_bidirectional.load()) +
	              ",csr_get_w_type_calls=" + std::to_string(g_calls_w_type.load()) +
	              ",reachability_calls=" + std::to_string(g_calls_reachability.load()) +
	              ",cheapest_path_calls=" + std::to_string(g_calls_cheapest_path.load()) +
	              ",shortest_path_count_calls=" + std::to_string(g_calls_path_count.load()) +
	              ",all_shortest_paths_calls=" + std::to_string(g_calls_all_shortest.load()) +
	              ",shortest_k_paths_calls=" + std::to_string(g_calls_shortest_k.load()) +
	              ",shortest_k_paths_mode_calls=" + std::to_string(g_calls_shortest_k_mode.load()) +
	              ",shortest_k_groups_calls=" + std::to_string(g_calls_shortest_k_groups.load()) +
	              ",shortest_k_groups_count_calls=" + std::to_string(g_calls_shortest_k_groups_count.load()) +
	              ",cheapest_path_count_calls=" + std::to_string(g_calls_cheapest_count.load()) +
	              ",all_cheapest_paths_calls=" + std::to_string(g_calls_all_cheapest.load()) +
	              ",cheapest_k_paths_calls=" + std::to_string(g_calls_cheapest_k.load());
	result.SetVectorType(VectorType::CONSTANT_VECTOR);
	ConstantVector::GetData<string_t>(result)[0] = StringVector::AddString(result, text);
}

int DuckpgqB200CompiledAbiVersion() {
	return PGQ_B200_ABI_VERSION;
}

void DuckpgqB200Extension::CheckAbi() {
	if (pgq_abi_version() != DuckpgqB200CompiledAbiVersion()) {
		throw InvalidInputException("duckpgq_b200: libduckpgq_b200.so speaks ABI version " +
		                            std::to_string(pgq_abi_version()) + ", this extension was built for " +
		                            std::to_string(DuckpgqB200CompiledAbiVersion()));
	}
}

// Re-registers every overload of a reference scalar function with `wrapper(reference callback, ...)` as its
// callback (same arguments, return type and bind, so the catalog replaces the overloads one by one).
typedef void (*wrapped_scalar_t)(const scalar_function_t &, DataChunk &, ExpressionState &, Vector &);
static void WrapScalar(ExtensionLoader &loader, const string &name, wrapped_scalar_t wrapper) {
	auto entry = loader.TryGetFunction(Identifier(name));
	if (!entry) {
		return; // (a reference build without this function)
	}
	ScalarFunctionSet wrapped {Identifier(name)};
	for (auto fun : entry->Cast<ScalarFunctionCatalogEntry>().functions.functions) { // (copies)
		scalar_function_t reference = fun.GetFunctionCallback();
		fun.SetFunctionCallback([reference, wrapper](DataChunk &args, ExpressionState &state, Vector &result) {
			wrapper(reference, args, state, result);
		});
		wrapped.AddFunction(std::move(fun));
	}
	loader.RegisterFunction(std::move(wrapped));
}

template <int K>
static void WrapTable(ExtensionLoader &loader, const string &name) {
	auto entry = loader.TryGetTableFunction(Identifier(name));
	if (!entry) {
		return;
	}
	auto &functions = entry->Cast<TableFunctionCatalogEntry>().functions.functions;
	if (functions.size() != 1) {
		return;
	}
	TableFunction fun = functions[0];
	TableWrap<K>::function = fun.function;
	TableWrap<K>::bind = fun.bind;
	fun.function = TableWrap<K>::Function;
	fun.bind = TableWrap<K>::Bind;
	TableFunctionSet set {Identifier(name)};
	set.AddFunction(std::move(fun));
	CreateTableFunctionInfo info(std::move(set));
	info.on_conflict = OnCreateConflict::REPLACE_ON_CONFLICT; // (ALTER only ADDS overloads to a table function)
	loader.RegisterFunction(std::move(info));
}

static void LoadInternal(ExtensionLoader &loader) {
	DuckpgqB200Extension::CheckAbi();
	// CSR construction: forward every chunk to the device build (the reference callbacks are captured)
	WrapScalar(loader, "create_csr_vertex", CreateCsrVertexB200);
	WrapScalar(loader, "create_csr_edge", CreateCsrEdgeB200);
	WrapScalar(loader, "delete_csr", DeleteCsrB200);
	WrapScalar(loader, "csr_get_w_type", CsrGetWTypeB200);
	// the other consumers of the CSR: on the device
	WrapScalar(loader, "local_clustering_coefficient", LocalClusteringCoefficientB200);
	WrapScalar(loader, "pagerank", PageRankB200);
	WrapScalar(loader, "weakly_connected_component", WeaklyConnectedComponentB200);
	WrapTable<0>(loader, "get_csr_v");
	WrapTable<1>(loader, "get_csr_e");
	WrapTable<2>(loader, "get_csr_w");
	WrapTable<3>(loader, "get_csr_ptr");
	// path functions: same names, argument types, return types and bind as the reference registrations
	// (iterativelength.cpp:148-152, shortest_path.cpp:212-217); bind = the reference's own
	// IterativeLengthBind (constant-folds the CSR id, marks it for deletion at bind time)
	loader.RegisterFunction(ScalarFunction(
	    "iterativelength", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::BIGINT, IterativeLengthB200Function, IterativeLengthFunctionData::IterativeLengthBind));
	loader.RegisterFunction(ScalarFunction(
	    "shortestpath", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::LIST(LogicalType::BIGINT), ShortestPathB200Function,
	    IterativeLengthFunctionData::IterativeLengthBind));
	// iterativelength2 (iterativelength2.cpp:13-31,139-141) is the same search with the `visit & ~seen[n]`
	// filter inside the edge loop -- exactly the formulation the top-down kernel uses; identical results
	loader.RegisterFunction(ScalarFunction(
	    "iterativelength2", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::BIGINT, IterativeLengthB200Function, IterativeLengthFunctionData::IterativeLengthBind));
	// iterativelengthbidirectional: signature and bind of iterativelength_bidirectional.cpp:158-163
	loader.RegisterFunction(ScalarFunction(
	    "iterativelengthbidirectional",
	    {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT}, LogicalType::BIGINT,
	    IterativeLengthBidirectionalB200Function, IterativeLengthFunctionData::IterativeLengthBind));
	// reachability: signature and bind of reachability.cpp:259-264
	loader.RegisterFunction(ScalarFunction(
	    "reachability",
	    {LogicalType::INTEGER, LogicalType::BOOLEAN, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::BOOLEAN, ReachabilityB200Function, IterativeLengthFunctionData::IterativeLengthBind));
	loader.RegisterFunction(ScalarFunction(
	    "cheapest_path_length", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::ANY, CheapestPathLengthB200Function, CheapestPathLengthFunctionData::CheapestPathLengthBind));
	// cheapest_path: no reference function is replaced; called as a raw UDF over the CSR CTE (the MATCH rewriter has
	// no CHEAPEST)
	loader.RegisterFunction(ScalarFunction(
	    "cheapest_path", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::LIST(LogicalType::BIGINT), CheapestPathB200Function, CheapestPathBind));
	// cheapest_path_count / all_cheapest_paths: ALL CHEAPEST's count and lists, raw UDFs like cheapest_path
	loader.RegisterFunction(ScalarFunction(
	    "cheapest_path_count", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::BIGINT, CheapestPathCountB200Function, CheapestPathCountBind));
	loader.RegisterFunction(ScalarFunction(
	    "all_cheapest_paths",
	    {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)), AllCheapestPathsB200Function, AllCheapestPathsBind));
	// cheapest_k_paths / cheapest_k_costs: CHEAPEST k's paths and their costs, raw UDFs like cheapest_path (5 arguments:
	// WALK; a 6th, VARCHAR mode)
	const vector<LogicalType> ck_args {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT,
	                                   LogicalType::BIGINT};
	vector<LogicalType> ck_mode_args = ck_args;
	ck_mode_args.push_back(LogicalType::VARCHAR);
	ScalarFunctionSet cheapest_k {Identifier("cheapest_k_paths")};
	for (auto &sig : {ck_args, ck_mode_args}) {
		cheapest_k.AddFunction(ScalarFunction(sig, LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)),
		                                      CheapestKPathsB200Function, CheapestKPathsBind));
	}
	loader.RegisterFunction(cheapest_k);
	ScalarFunctionSet cheapest_k_costs {Identifier("cheapest_k_costs")};
	for (auto &sig : {ck_args, ck_mode_args}) {
		cheapest_k_costs.AddFunction(ScalarFunction(sig, LogicalType::ANY, CheapestKCostsB200Function, CheapestKCostsBind));
	}
	loader.RegisterFunction(cheapest_k_costs);
	// shortest_path_count / all_shortest_paths: no reference function is replaced; raw UDFs over the CSR CTE (the
	// reference's MATCH rewriter rejects ALL SHORTEST)
	loader.RegisterFunction(ScalarFunction(
	    "shortest_path_count", {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::BIGINT, ShortestPathCountB200Function, IterativeLengthFunctionData::IterativeLengthBind));
	loader.RegisterFunction(ScalarFunction(
	    "all_shortest_paths",
	    {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)), AllShortestPathsB200Function, AllShortestPathsBind));
	// shortest_k_paths: the walks (5 arguments) and SQL/PGQ's path modes (a 6th, VARCHAR mode)
	ScalarFunctionSet shortest_k {Identifier("shortest_k_paths")};
	shortest_k.AddFunction(ScalarFunction(
	    {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	    LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)), ShortestKPathsB200Function, ShortestKPathsBind));
	shortest_k.AddFunction(ScalarFunction({LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT,
	                                       LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::VARCHAR},
	                                      LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT)),
	                                      ShortestKPathsModeB200Function, ShortestKPathsModeBind));
	loader.RegisterFunction(shortest_k);
	// shortest_k_groups: SHORTEST k GROUP's paths (6 arguments: WALK; a 7th, VARCHAR mode) and WALK's count
	const auto lists = LogicalType::LIST(LogicalType::LIST(LogicalType::BIGINT));
	ScalarFunctionSet shortest_k_groups {Identifier("shortest_k_groups")};
	shortest_k_groups.AddFunction(ScalarFunction({LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT,
	                                              LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT},
	                                             lists, ShortestKGroupsB200Function, ShortestKGroupsBind));
	shortest_k_groups.AddFunction(ScalarFunction({LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT,
	                                              LogicalType::BIGINT, LogicalType::BIGINT, LogicalType::BIGINT,
	                                              LogicalType::VARCHAR},
	                                             lists, ShortestKGroupsB200Function, ShortestKGroupsBind));
	loader.RegisterFunction(shortest_k_groups);
	loader.RegisterFunction(ScalarFunction("shortest_k_groups_count",
	                                       {LogicalType::INTEGER, LogicalType::BIGINT, LogicalType::BIGINT,
	                                        LogicalType::BIGINT, LogicalType::BIGINT},
	                                       LogicalType::BIGINT, ShortestKGroupsCountB200Function, ShortestKPathsBind));
	ScalarFunction stats("duckpgq_b200_stats", {}, LogicalType::VARCHAR, B200StatsFunction);
	stats.SetVolatile();
	loader.RegisterFunction(stats);
}

void DuckpgqB200Extension::Load(ExtensionLoader &loader) {
	LoadInternal(loader);
}

std::string DuckpgqB200Extension::Name() {
	return "duckpgq_b200";
}

} // namespace duckdb

extern "C" {

DUCKDB_CPP_EXTENSION_ENTRY(duckpgq_b200, loader) {
	duckdb::LoadInternal(loader);
}
}
