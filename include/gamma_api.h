/*
 * gamma_api.h -- the gamma engine C-ABI, re-exported by the H100-native libgamma.so.
 *
 * Drop-in boundary (SURVEY.md 8b): these are exactly the 23 entry points the Go partition
 * server binds through cgo (`#cgo LDFLAGS: -lgamma`, internal/engine/sdk/go/gamma/gamma.go:10-17)
 * with the signatures of the reference header internal/engine/c_api/gamma_api.h:15-188 and the
 * behaviour of internal/engine/c_api/gamma_api.cc:35-374.  Payload encodings are the
 * reference's: JSON (Init / SetConfig / status), flatbuffers gamma_api.Table / gamma_api.Doc
 * (idl/fbs/table.fbs, doc.fbs), protobuf vearchpb.SearchRequest / SearchResponse
 * (internal/proto/router_grpc.proto:168-219).
 *
 * Ownership: inputs are borrowed for the duration of the call; every char** output and every
 * non-NULL CStatus.msg is malloc()'d here and free()'d by the caller (the Go side calls C.free,
 * gamma.go:47-53,78-81,176-181).  CStatus.code is vearch::status::Code (idl/fbs/status.fbs):
 * 0 ok, 1 not found, 2 index error, 3 not supported, 4 invalid argument, 5 IO error, 6 busy,
 * 7 timed out, 8 memory exceeded, 9 cancelled.
 *
 * Scope of this build (DESIGN.md, INTEGRATION.md): full semantics for Init / Close / CreateTable /
 * AddOrUpdateDoc / DeleteDoc / GetDocByID / GetDocByDocID / BuildIndex / Search / Query /
 * GetEngineStatus / GetMemoryInfo / SetConfig / GetConfig / Dump / Load / Backup / SetKillStatus /
 * DeleteKillStatus / AddFieldIndexWithParams / RemoveFieldIndex / RebuildIndex / SetMemoryLimitConfig for
 * tables whose vector fields are indexed as FLAT, IVFFLAT or IVFPQ (optionally with OPQ).  Backup(engine, 0) writes
 * what Dump writes into <path>/backup/retrieval_model_index, captured on the device under the table lock and written
 * after it is released; Backup(engine, 1) does nothing.  SetMemoryLimitConfig(p) limits what this library holds to p % of each device's HBM and of host
 * memory (0: no limit): past it AddOrUpdateDoc refuses new documents with -5 and Search / Query return code 8.
 */
#ifndef GAMMA_API_H_
#define GAMMA_API_H_

#ifdef __cplusplus
extern "C" {
#endif

struct CStatus {
  int code;
  char *msg;
};

/* gamma_api.cc:35-70.  config JSON: {"path": ..., "space_name": ..., "log_dir": ...,
 * optional "device": GPU ordinal (default 0; partitions map to GPUs, SURVEY.md 8e),
 * optional "devices": GPU ordinals [0, 1, ...] or "all": GPU_IVFPQ / GPU_IVFFLAT fields are sharded over them and
 * devices[0] replaces "device"; an ordinal outside the visible devices makes Init return NULL}.
 * The environment variables GAMMA_B200_DEVICE and GAMMA_B200_DEVICES ("0,1,2,3" or "all") override the two keys.
 * Returns NULL on failure (gammacb/gamma.go:84-88). */
void *Init(const char *config_str, int len);
/* gamma_api.cc:137-141 */
int Close(void *engine);
/* gamma_api.cc:156-166; table_str = flatbuffers gamma_api.Table */
struct CStatus CreateTable(void *engine, const char *table_str, int len);
/* gamma_api.cc:168-173; doc_str = flatbuffers gamma_api.Doc; 0 ok, -1..-7 by failing stage
 * (search/engine.cc:704-751) */
int AddOrUpdateDoc(void *engine, const char *doc_str, int len);
/* gamma_api.cc:229-233; -1 = unknown key */
int DeleteDoc(void *engine, const char *docid, int docid_len);
/* gamma_api.cc:273-278; JSON {index_status, backup_status, doc_num, max_docid, min_indexed_num} */
void GetEngineStatus(void *engine, char **status, int *len);
/* gamma_api.cc:280-286; JSON {table_mem, index_mem, vector_mem, field_range_mem, bitmap_mem} */
void GetMemoryInfo(void *engine, char **memory_info, int *len);
/* gamma_api.cc:235-242 / 244-255; doc_str = flatbuffers gamma_api.Doc */
int GetDocByID(void *engine, const char *docid, int docid_len, char **doc_str, int *len);
int GetDocByDocID(void *engine, int docid, char next, char **doc_str, int *len);
/* gamma_api.cc:257-260; returns immediately, training + indexing continue on an engine thread
 * (search/engine.cc:951-988) */
int BuildIndex(void *engine);
int RebuildIndex(void *engine, int drop_before_rebuild, int limit_cpu, int describe);
/* gamma_api.cc:288-296 */
int Dump(void *engine);
int Load(void *engine);
/* gamma_api.cc:174-201; request_str = protobuf vearchpb.SearchRequest, *response_str =
 * protobuf vearchpb.SearchResponse */
struct CStatus Search(void *engine, const char *request_str, int req_len, char **response_str, int *res_len);
struct CStatus Query(void *engine, const char *request_str, int req_len, char **response_str, int *res_len);
/* gamma_api.cc:298-311; JSON {engine_cache_size, slow_search_time, refresh_interval, enable_id_cache} */
int SetConfig(void *engine, const char *config_str, int len);
int GetConfig(void *engine, char **config_str, int *len);
struct CStatus Backup(void *engine, int command);
struct CStatus AddFieldIndexWithParams(void *engine, const char *field_name, int field_name_len,
                                       const char *index_type, int index_type_len, const char *index_params,
                                       int index_params_len);
struct CStatus RemoveFieldIndex(void *engine, const char *field_name, int field_name_len);
/* gamma_api.cc:352-374.  memory_limit: percent of each device's total HBM and of host memory this process's library
 * allocations may hold (DESIGN.md section 8); 0 removes the limit */
void SetMemoryLimitConfig(int memory_limit);
void SetKillStatus(const char *request_id, int partition_id, int reason);
void DeleteKillStatus(const char *request_id, int partition_id);

#ifdef __cplusplus
}
#endif
#endif /* GAMMA_API_H_ */
