# DuckDB extension list for the combined build: the UNMODIFIED reference first, then the GPU
# override (LoadAllExtensions loads in list order, duckdb/extension/generated_extension_loader.cpp.in:14-26).
if(NOT DEFINED PGQ_REFERENCE_DIR)
  set(PGQ_REFERENCE_DIR "/root/reference")
endif()
duckdb_extension_load(duckpgq
    SOURCE_DIR ${PGQ_REFERENCE_DIR}
)
duckdb_extension_load(duckpgq_b200
    SOURCE_DIR ${CMAKE_CURRENT_LIST_DIR}
)
