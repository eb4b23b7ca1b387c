/* llmgw_b200 -- C ABI of the H100 streaming chat-completions transform engine.
 *
 * Drop-in boundary for the per-request hot path of fabiojbg/LLMApiGateway (SURVEY.md 8(b)).
 * The reference exposes no FFI for this path (it is inline Python); each entry point below
 * names the reference code whose per-byte work it replaces.  Paths are relative to the
 * reference root.  INTEGRATION.md shows the ctypes binding a maintainer adds on the Python side.
 *
 * Conventions
 *   - plain pointers and sizes only; the caller owns every buffer it passes in;
 *   - every function returns 0 on success or a negative lgw_status; nothing throws across the
 *     boundary; lgw_last_error() gives a human-readable reason;
 *   - data errors (bad JSON, failed attempt, ...) are VALUES in the outputs, like the
 *     reference's (None, error_detail) returns -- never a non-zero status;
 *   - there is no CPU fallback: without a CUDA device lgw_engine_create fails;
 *   - an engine handle is not thread-safe (one batcher thread per GPU owns it).
 */
#ifndef LLMGW_B200_H
#define LLMGW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LGW_ABI_VERSION 1

typedef enum lgw_status {
    LGW_OK = 0,
    LGW_ERR_ARG = -1,        /* bad argument (null pointer, unsorted offsets, unknown slot ...) */
    LGW_ERR_CUDA = -2,       /* a CUDA runtime call failed */
    LGW_ERR_CAPACITY = -3,   /* step larger than the limits given at create time */
    LGW_ERR_NO_DEVICE = -4   /* no usable CUDA device: the engine never computes on the CPU */
} lgw_status;

/* ---- value model ---------------------------------------------------------------------------
 * JSON values copied "untyped" by chat_logging.py:248-267 keep their Python type, so every
 * extracted field is a tagged value. */
enum lgw_kind {
    LGW_KIND_ABSENT = 0, LGW_KIND_INT = 1, LGW_KIND_FLOAT = 2, LGW_KIND_NULL = 3, LGW_KIND_TRUE = 4,
    LGW_KIND_FALSE = 5, LGW_KIND_STR = 6, LGW_KIND_BIGINT = 7, LGW_KIND_OBJECT = 8, LGW_KIND_ARRAY = 9,
    LGW_KIND_FLOAT_INEXACT = 10
};

typedef struct lgw_val {
    int64_t bits;            /* INT: the value; FLOAT: IEEE-754 binary64 bit pattern */
    uint8_t kind;            /* enum lgw_kind */
    uint8_t _pad[7];
} lgw_val;

#define LGW_STR_CAP 120

/* The dict get_token_usage returns (chat_logging.py:233-272), after its reasoning-token
 * subtraction (:262-263).  model_val/provider_val.kind == ABSENT means the key is not in the dict. */
typedef struct lgw_usage_rec {
    lgw_val prompt_tokens, completion_tokens, total_tokens, reasoning_tokens, cached_tokens, cost;
    lgw_val model_val, provider_val;
    uint8_t model_len, provider_len;
    uint8_t str_flags;       /* bit0/1: model truncated / lone surrogate; bit2/3: provider */
    uint8_t exotic;          /* 1: some value is not representable here (big int, string where a number goes ...) */
    char model[LGW_STR_CAP];
    char provider[LGW_STR_CAP];
} lgw_usage_rec;

/* stream phases and verdicts (request_handler.py:65-98) */
enum lgw_phase { LGW_PHASE_FREE = 0, LGW_PHASE_PRIMING = 1, LGW_PHASE_COMMITTED = 2, LGW_PHASE_FAILED = 3 };
enum lgw_verdict {
    LGW_VERDICT_NONE = 0,
    LGW_VERDICT_OK = 1,          /* first real event accepted (:89-90) */
    LGW_VERDICT_FAIL_EVENT = 2,  /* first real event carries top-level "error"/"detail" (:50-54,:86-88) */
    LGW_VERDICT_FAIL_PARSE = 3,  /* first real event is not JSON (:85 -> :183-187) */
    LGW_VERDICT_FAIL_HTTP = 4    /* upstream status >= 400 (:25-30) */
};
enum lgw_stream_flag {
    LGW_SF_A_USAGE_BOUND = 1 << 0,   /* request_handler.py:134 ran (otherwise :144 raises UnboundLocalError) */
    LGW_SF_EMITTED_ANY = 1 << 1,     /* a chunk was relayed => a tap thread / DB row exists (chat_logging.py:200) */
    LGW_SF_CARRY_OVERFLOW = 1 << 2,  /* an unterminated event outgrew carry_cap (engine limit, reported) */
    LGW_SF_EXOTIC_SEEN = 1 << 3,
    LGW_SF_SYNCED = 1 << 4,
    LGW_SF_REC_VALID = 1 << 5,
    LGW_SF_DETAIL_TRUNC = 1 << 6,
    LGW_SF_ROWQ_OVERFLOW = 1 << 7,
    LGW_SF_PENDING = 1 << 8          /* internal: usage event stashed, extracted when the state is read */
};

typedef struct lgw_stream_state {
    uint8_t phase, verdict;
    uint16_t flags;
    uint32_t carry_a_len, carry_b_len, detail_len;
    uint32_t n_events_a, n_events_b, n_usage_b, n_exotic, n_error_rows;
    uint32_t n_chunks_in, n_chunks_emitted;
    uint32_t pending_len;        /* internal (see LGW_SF_PENDING); always 0 in states returned to the host */
    uint64_t bytes_in, bytes_emitted;
    lgw_usage_rec rec;       /* current tap record (valid when LGW_SF_REC_VALID, else the defaults) */
} lgw_stream_state;

/* a write_log call that happened mid-stream: tap saw a top-level "error" (chat_logging.py:137-139) */
typedef struct lgw_row_event {
    uint32_t slot, seq;
    lgw_usage_rec rec;
} lgw_row_event;

typedef struct lgw_seg_result {
    uint32_t emit_chunk_begin;   /* first chunk of the segment that is relayed this step; the relayed
                                    chunks are [emit_chunk_begin, segment end): always a suffix */
    uint8_t phase, verdict;
    uint16_t flags;
    uint32_t detail_len;         /* > 0 with a FAIL_* verdict: fetch with lgw_stream_detail */
} lgw_seg_result;

typedef struct lgw_limits {
    uint32_t max_streams;        /* stream slots resident on the device */
    uint32_t carry_cap;          /* bytes of unterminated event kept per stream between steps */
    uint32_t detail_cap;         /* bytes of error detail kept per stream */
    uint32_t rowq_cap;           /* mid-stream row events per step */
    uint32_t max_step_chunks;    /* chunks per step (host-buffer entry points stage this much) */
    uint64_t max_step_bytes;     /* bytes per step */
} lgw_limits;

typedef struct lgw_engine lgw_engine;

/* ---- lifetime --------------------------------------------------------------------------------- */
int lgw_abi_version(void);
int lgw_engine_create(int device, const lgw_limits* limits, lgw_engine** out);
int lgw_engine_destroy(lgw_engine* e);
const char* lgw_last_error(const lgw_engine* e);    /* e may be NULL: error of the last failed create */
/* run on a caller-owned cudaStream_t (e.g. torch's current stream); NULL = the engine's own stream */
int lgw_engine_set_stream(lgw_engine* e, void* cuda_stream);

/* ---- streams ------------------------------------------------------------------------------------
 * One slot = one upstream attempt of make_llm_request(..., is_streaming=True)
 * (llm_gateway_core/services/request_handler.py:8).  http_status is the upstream response status
 * (:25-30): >= 400 marks the attempt failed at once and the host keeps the body as error detail.
 * Stream-ordered on the engine stream: returns without waiting for the GPU; the arrays are copied
 * before it returns, so the caller may reuse them at once. */
int lgw_streams_open(lgw_engine* e, const uint32_t* slots, const int32_t* http_status, uint32_t n);
int lgw_streams_state(lgw_engine* e, const uint32_t* slots, uint32_t n, lgw_stream_state* out);
/* error detail of a failed attempt: the text the reference stores at request_handler.py:51,87
 * (the whole first event, "data: " included) */
int lgw_stream_detail(lgw_engine* e, uint32_t slot, uint8_t* buf, uint32_t cap, uint32_t* len);
/* the same for n slots in one round trip (config 4: the failed attempts of a round): slot i's text is
 * buf[i*stride .. i*stride + lens[i]), cut at `stride` bytes */
int lgw_streams_details(lgw_engine* e, const uint32_t* slots, uint32_t n, uint8_t* buf, uint32_t stride, uint32_t* lens);
/* end of upstream: final state (the last DB row of chat_logging.py:150 is `rec` when
 * LGW_SF_EMITTED_ANY), slot returns to FREE */
int lgw_streams_close(lgw_engine* e, const uint32_t* slots, uint32_t n, lgw_stream_state* final_out);

/* ---- the hot path ---------------------------------------------------------------------------------
 * One batched pass over the newly arrived upstream chunks of many streams.  Replaces, per chunk,
 *   request_handler.py:34-63   stream_generator   (decode, split on "\n\n", "data: {" test, first-event sniff)
 *   request_handler.py:69-98   priming loop        (keep/drop, error/detail verdict)
 *   request_handler.py:109-142 combined_generator  (parse, "code"/"usage" keys, relay bytes)
 *   chat_logging.py:90-147     ChunkProcessorThread.run (parse again, choices walk, usage extraction)
 *   chat_logging.py:233-272    get_token_usage
 *
 * Layout: chunk_bytes holds every chunk back to back; chunk c is bytes [chunk_off[c], chunk_off[c+1]).
 * Chunks are grouped per stream in arrival order: segment s is chunks [seg_chunk[s], seg_chunk[s+1])
 * of stream slot seg_slot[s]; a slot appears in at most one segment per step.
 *
 * out_bytes (same size as chunk_bytes) receives the re-emitted stream: for every relayed chunk
 * the bytes at the same offsets (the reference relays original bytes, :141-142); bytes of dropped
 * chunks are unspecified.  seg_out[s].emit_chunk_begin says where relaying starts in segment s.
 * rows_out/n_rows: mid-stream row events of this step, in no particular order across streams
 * (seq orders them within a stream).
 *
 * out_bytes may be NULL in lgw_sse_step ("verdicts only"): the relayed bytes are by construction the caller's own bytes at the
 * same offsets, so a caller that keeps its chunks (the batcher does) can relay those and save the download; everything else
 * (seg_out, rows, stream state, the device-side re-emit) is unchanged.
 *
 * lgw_sse_step takes HOST pointers and performs the H2D/D2H copies itself (synchronous).
 * lgw_sse_step_device takes DEVICE pointers for the five input arrays and out_bytes/seg_out, is
 * asynchronous on the engine stream, and leaves row events on the device until lgw_fetch_rows. */
int lgw_sse_step(lgw_engine* e,
                 const uint8_t* chunk_bytes, uint64_t n_bytes,
                 const uint32_t* chunk_off, uint32_t n_chunks,
                 const uint32_t* seg_chunk, const uint32_t* seg_slot, uint32_t n_segs,
                 uint8_t* out_bytes, lgw_seg_result* seg_out,
                 lgw_row_event* rows_out, uint32_t rows_cap, uint32_t* n_rows);
int lgw_sse_step_device(lgw_engine* e,
                        const uint8_t* d_chunk_bytes, uint64_t n_bytes,
                        const uint32_t* d_chunk_off, uint32_t n_chunks,
                        const uint32_t* d_seg_chunk, const uint32_t* d_seg_slot, uint32_t n_segs,
                        uint8_t* d_out_bytes, lgw_seg_result* d_seg_out);
int lgw_fetch_rows(lgw_engine* e, lgw_row_event* rows_out, uint32_t rows_cap, uint32_t* n_rows);
int lgw_sync(lgw_engine* e);

/* device time of the kernels of the last step (CUDA events on the launching stream), milliseconds:
 * [0] prime  [1] relay (bulk parse + re-emit)  [2] commit (incl. usage extraction)  [3] whole step incl. copies (host entry only);
 * see lgw_last_step_kernel_ms for what [0..2] hold when the kernels overlap */
int lgw_last_step_ms(lgw_engine* e, float ms[4]);
/* the kernels one by one: [0] prime  [1] relay  [2] commit  [3] 0 (usage extraction happens inside relay and commit).
 * By default the kernels of a step are chained with programmatic dependent launches (each one's prologue overlaps the one
 * before): then only their total is meaningful and comes back in [1].  lgw_engine_set_kernel_timing(e, 1) puts CUDA events
 * between them instead (back-to-back launches) for a per-kernel breakdown. */
int lgw_last_step_kernel_ms(lgw_engine* e, float ms[4]);
int lgw_engine_set_kernel_timing(lgw_engine* e, int on);
/* number of kernels launched by this engine since creation */
/* 1 when the last lgw_sse_step ran in direct mode: both byte buffers were page-locked host memory and the bulk kernel moved
 * them over PCIe itself (TMA loads from / stores to the host buffers), without the staged, sliced copies */
int lgw_last_step_direct(lgw_engine* e);
int lgw_launch_count(lgw_engine* e, uint64_t* out);

/* ---- usage-stats rollup -----------------------------------------------------------------------------
 * Replaces the scan inside TokensUsageDB.get_aggregated_usage (llm_gateway_core/db/tokens_usage_db.py:222-304,
 * SQL at :268-286): GROUP BY strftime(fmt, timestamp), model; SUM of the five token columns, SUM(cost),
 * COUNT(*); optional window on timestamp (:255-266).  Records are device-resident SoA columns
 * (40 B per record): ts_us = microseconds of the naive local timestamp the reference stores
 * (:135), model_rank = 0 for NULL else 1 + rank of the model name in byte order.
 * period: 0 hour, 1 day, 2 week ('%Y-W%W'), 3 month.  Bucket numbering: see lgw_rollup_row.bucket.
 *
 * lgw_usage_rollup_accum adds the records into a dense table of 64-bit integer cells
 * [n_buckets][n_models][LGW_ROLLUP_CELLS] (d_table, zeroed by the caller) -- every cell is an
 * integer sum, so tables from several GPUs merge with an element-wise add (ncclAllReduce sum) --
 * and lgw_usage_rollup_emit turns a table into rows ordered like the SQL (time_period DESC, model ASC). */
#define LGW_ROLLUP_CELLS 10
typedef struct lgw_rollup_row {
    int64_t bucket;          /* hour: hours since 1970-01-01T00; day: days since 1970-01-01;
                                week: year*64 + %W; month: year*12 + month-1 */
    int32_t model_rank;
    uint32_t inexact;        /* 1: some cost in the group was not taken exactly (bits below 2^-80, |cost| >= 2^12,
                                NaN = NULL, +-Inf): `cost` is not the group's sum, the caller sums it again */
    int64_t prompt_tokens, completion_tokens, total_tokens, reasoning_tokens, cached_tokens;
    double cost;
    int64_t count;
} lgw_rollup_row;

int lgw_usage_rollup_accum(lgw_engine* e, const int64_t* d_ts_us, const int32_t* d_model_rank,
                           const int32_t* d_prompt, const int32_t* d_completion, const int32_t* d_total,
                           const int32_t* d_reasoning, const int32_t* d_cached, const double* d_cost, uint64_t n,
                           int period, int has_start, int64_t start_us, int has_end, int64_t end_us,
                           int64_t bucket0, uint32_t n_buckets, uint32_t n_models,
                           uint64_t* d_table, uint32_t* d_inexact, uint32_t* d_out_of_table);
int lgw_usage_rollup_emit(lgw_engine* e, const uint64_t* d_table, const uint32_t* d_inexact,
                          int64_t bucket0, uint32_t n_buckets, uint32_t n_models,
                          lgw_rollup_row* rows_out /* host */, uint64_t rows_cap, uint64_t* n_rows);
/* bucket index of one timestamp (host helper, same arithmetic as the kernel) */
int64_t lgw_rollup_bucket_of(int64_t ts_us, int period);
/* the same for n timestamps (host memory); 0 or LGW_ERR_ARG */
int lgw_rollup_buckets_of(const int64_t* ts_us, uint64_t n, int period, int64_t* out);
/* device time of the last accum / emit kernels, milliseconds */
/* accumulate path: 0 (default) block-privatised shared-memory tables whenever bucket x model groups <= 2560 (every window
 * the stats endpoint asks for, stats.py:46-55), global 64-bit reductions else; 1 forces the global path (tests, measurements) */
int lgw_rollup_set_path(lgw_engine* e, int force_global);
int lgw_rollup_last_ms(lgw_engine* e, float ms[2]);

/* /v1/api/usage-records (tokens_usage_db.py:69-117): the record indices at ranks [first, first + count) of the order
 * (ts_us DESC, index ASC) over n device-resident timestamps; idx_out is host memory.  n >= 2^32 or first + count > n: LGW_ERR_ARG
 * (so is a d_ts_us that is not 16-byte aligned; cudaMalloc memory is).  Equal timestamps list in index (insertion) order.
 * Device work: a radix select of the keys at both ends of the page (12 passes of 8-bit digits over the timestamp and the
 * index; the passes read only the candidates once they are at most n/16), one ordered compaction of the page, and a sort of
 * it: in one block up to 8192 records, a stable LSD radix sort above (csrc/listing.cuh).  count == 0 launches nothing. */
int lgw_usage_latest(lgw_engine* e, const int64_t* d_ts_us, uint64_t n, uint64_t first, uint64_t count, uint64_t* idx_out);
/* device time of the last lgw_usage_latest, milliseconds (0 after a call with count == 0) */
int lgw_usage_latest_last_ms(lgw_engine* e, float* ms);

/* cleanup_old_records (tokens_usage_db.py:164-198, `DELETE FROM tokens_usage WHERE timestamp < ?`): the n device-resident
 * records whose ts_us >= cutoff_us, written in index order (a stable compaction) into the fresh columns d_out.  d_in / d_out
 * hold the eight column pointers in UsageTable.COLS order: ts_us (int64), model_rank, prompt, completion, total, reasoning,
 * cached (int32), cost (double); d_out has room for n_keep records per column and must not overlap d_in.  n_keep is the survivor
 * count the caller computed; only places below it are written, and a device count that differs fails the call (LGW_ERR_CUDA,
 * message in lgw_last_error) with nothing written past the output.  n >= 2^32, n_keep > n, a null pointer when n > 0 (d_out
 * may be null when n_keep == 0) or a d_in[0] that is not 16-byte aligned: LGW_ERR_ARG.  n == 0 launches nothing.
 * Device work: k_retain_count, k_list_scan, k_retain_write (csrc/retain.cuh). */
int lgw_usage_retain(lgw_engine* e, void* const d_in[8], void* const d_out[8], uint64_t n, int64_t cutoff_us, uint64_t n_keep);
/* device time of the last lgw_usage_retain, milliseconds (0 after a call with n == 0) */
int lgw_usage_retain_last_ms(lgw_engine* e, float* ms);

/* insert_usage (tokens_usage_db.py:119-162) on the device copy: m new records appended after the n resident ones.  Columns in
 * UsageTable.COLS order, typed as lgw_usage_retain's.  d_cols holds the n resident records; h_new the m new ones in host
 * memory, their model_rank final.  d_grow == NULL: the new rows go to d_cols[c] + n (the caller guarantees room for n + m);
 * else d_grow are fresh columns with room for n + m, not overlapping d_cols, and records [0, n) are copied into them first.
 * rank_map (host, n_map entries, or NULL): a resident record's model_rank r becomes rank_map[r], in place or while it is
 * copied.  A resident rank >= n_map (or negative) is counted on the device and fails the call (LGW_ERR_CUDA, message in
 * lgw_last_error); that record keeps its rank.  Nothing is written outside [0, n + m) of the target columns.  n + m >= 2^32,
 * a null pointer that the call needs, a ts_us column (d_cols or d_grow) that is not 16-byte aligned, or rank_map with
 * n_map == 0: LGW_ERR_ARG.  m == 0 with neither a map nor d_grow launches nothing.
 * Device work: one host-to-device copy of the new rows and the map through engine-owned page-locked staging, and one launch of
 * k_usage_append (csrc/append.cuh).  The call returns when the columns are written. */
int lgw_usage_append(lgw_engine* e, void* const d_cols[8], void* const d_grow[8], uint64_t n,
                     const void* const h_new[8], uint64_t m, const int32_t* rank_map, uint32_t n_map);
/* device time of the last lgw_usage_append (its copy and kernel), milliseconds (0 after a call that launched nothing) */
int lgw_usage_append_last_ms(lgw_engine* e, float* ms);

/* ---- loading the usage table from a `tokens_usage` SQLite file (tokens_usage_db.py:37-50) ------------------------------------
 * Four calls, in order, on one engine (csrc/load.cuh):
 * lgw_usage_load_decode: copies pages [1, n_pages] of h_file (page-locked host memory, n_bytes >= n_pages * page_size) to the
 *   device in one copy, walks the table b-tree from page `root`, decodes every record and builds the model / provider
 *   dictionaries.  out[6] = {LoadError (0: none; the rest of out is then meaningless), records, distinct model texts, distinct
 *   provider texts, their total bytes (model, provider)}.  A page size that is not a power of two in [512, 65536], n_pages == 0
 *   or too large for n_bytes, or n_bytes >= 2^33: LGW_ERR_ARG.  The file's own header is the caller's to check.
 * lgw_usage_load_names: the distinct texts of `field` (0 model, 1 provider) in provisional-code order, read from h_file (the
 *   buffer given to decode): buf holds out[4 + field] bytes, offs out[2 + field] + 1 offsets.
 * lgw_usage_load_mark: maps (provisional code -> anything >= 0, or -1: refuse every record with that text) for both fields;
 *   model_used[code] = 1 for each model text a kept record has; *n_keep = the records kept.
 * lgw_usage_load_finish: the kept records in rowid order into d_cols (the eight UsageTable.COLS columns, n_keep records each,
 *   caller-allocated) and into h_cols, with ids into h_ids, provider codes (prov_map[code], 0 for NULL) into h_prov; the ids of
 *   the other records into h_refused.  model_map now gives ranks (0 for NULL); both maps must refuse what they refused in mark
 *   (else LGW_ERR_ARG).  A call out of order: LGW_ERR_ARG.
 * The load's device scratch (the file, per-record arrays, dictionaries) lives only from decode to the end of finish, or to a
 * decode that found damage; lgw_usage_load_release frees it at any point (a load abandoned between the calls) and waits for
 * the engine stream first.  A load is used once, at startup: nothing of it stays on the device but the caller's columns. */
int lgw_usage_load_decode(lgw_engine* e, const uint8_t* h_file, uint64_t n_bytes, uint32_t page_size, uint32_t n_pages, uint32_t root, uint64_t out[6]);
int lgw_usage_load_names(lgw_engine* e, const uint8_t* h_file, int field, uint8_t* buf, uint64_t* offs);
int lgw_usage_load_mark(lgw_engine* e, const int32_t* model_map, const int32_t* prov_map, uint8_t* model_used, uint64_t* n_keep);
int lgw_usage_load_finish(lgw_engine* e, const int32_t* model_map, const int32_t* prov_map, void* const d_cols[8], void* const h_cols[8],
                          int64_t* h_ids, int32_t* h_prov, int64_t* h_refused);
int lgw_usage_load_release(lgw_engine* e);
/* device times of the last load, milliseconds: {host-to-device copy, b-tree walk and record decode, dictionaries, mark and finish} */
int lgw_usage_load_last_ms(lgw_engine* e, float ms[4]);

/* ---- saving the usage table as a `tokens_usage` SQLite file (the file lgw_usage_load_* reads) --------------------------------
 * Two calls, in order, on one engine (csrc/save.cuh):
 * lgw_usage_save_plan: the n records of d_cols (the eight UsageTable.COLS device columns, ts_us 16-byte aligned) with their ids
 *   (h_ids, ascending) and provider codes (h_prov), host memory copied up for the call.  Text tables: text k of `models` is
 *   model rank k, of `providers` provider code k; len[k] is its byte count, LGW_SAVE_TEXT_NULL for NULL or LGW_SAVE_TEXT_BAD
 *   for a text the file cannot hold; off has n + 1 entries, off[n] the blob's size.  A record is kept unless a text of it is
 *   BAD or its ts_us has no datetime.isoformat() text (years 0001-9999).  Lays out the file for page_size (a power of two in
 *   [1024, 65536]): out[5] = {pages of the whole file, table root page, index root page, kept records, refused records}.
 *   Pages 1 (header and sqlite_schema) and 2 (sqlite_sequence) are the caller's.  LGW_ERR_ARG: n >= 2^32, a null pointer the
 *   call needs, a misaligned ts_us column, an empty text table, a rank or code outside its table, ids not ascending, or a
 *   file of 2^32 - 1 pages or more.
 * lgw_usage_save_write: pages 3 .. out[0] into h_file + 2 * page_size (page-locked, out[0] * page_size bytes), the refused
 *   records' ids in record order into h_refused (out[4] entries).
 * The save's device scratch (ids and codes, per-record arrays, the page pool, the file image) lives only from plan to the end
 * of write; lgw_usage_save_release frees it at any point and waits for the engine stream first. */
typedef struct lgw_save_text { const uint8_t* blob; const uint64_t* off; const uint32_t* len; uint32_t n, pad; } lgw_save_text;
#define LGW_SAVE_TEXT_NULL 0xFFFFFFFFu
#define LGW_SAVE_TEXT_BAD 0xFFFFFFFEu
int lgw_usage_save_plan(lgw_engine* e, void* const d_cols[8], uint64_t n, const int64_t* h_ids, const int32_t* h_prov,
                        const lgw_save_text* models, const lgw_save_text* providers, uint32_t page_size, uint64_t out[5]);
int lgw_usage_save_write(lgw_engine* e, uint8_t* h_file, int64_t* h_refused);
int lgw_usage_save_release(lgw_engine* e);
/* device times of the last save, milliseconds: {ids and codes up, keep, sort, pack, page writes, download} */
int lgw_usage_save_last_ms(lgw_engine* e, float ms[6]);

/* ---- request-body rewrite: SURVEY 8 rows a1, a3, a4 --------------------------------------------------
 * Replaces, for a batch of client requests, chat.py:31-45 (parse: lgw_bodies_scan) and, per upstream
 * attempt, chat.py:112-119,:135-139,:150,:164-168 (deepcopy + key assignments) followed by the encoder
 * of request_handler.py:23 (httpx `json=`) or :153 (json5.dumps): lgw_bodies_rewrite.
 * The rule table (loader.py:150-154 dicts) is compiled on the host into "plans": one plan = the ordered
 * key assignments of one attempt (rule x sub-provider x retry) in one render mode, with keys and values
 * already rendered (llmapigateway_b200/rewrite.py does this; rule lookup/rotation a2 stays in Python). */
enum lgw_render_mode {
    LGW_RM_HTTPX028 = 0,   /* json.dumps(ensure_ascii=False, separators=(",",":"), allow_nan=False)  (installed httpx 0.28.1) */
    LGW_RM_HTTPX027 = 1,   /* json.dumps(obj) stdlib defaults                                        (requirements.txt pin)   */
    LGW_RM_JSON5 = 2       /* json5.dumps defaults (non-streaming branch); restated, unpinned                               */
};
enum lgw_body_status {
    LGW_BODY_OK = 0,
    LGW_BODY_PARSE_ERROR = 1,   /* chat.py:37-39: HTTP 400 "Error reading request body" (bad UTF-8/JSON, not an object, no "model") */
    LGW_BODY_NO_MODEL = 2,      /* chat.py:44-45: HTTP 400 "Missing 'model'"                                                       */
    LGW_BODY_OVERFLOW = 3,      /* out slot too small: out_len holds the size needed                                               */
    LGW_BODY_EXOTIC = 4,        /* shape the engine does not model (duplicate keys, float with > 15 significant digits,
                                   key > 128 B, > 24 keys in one object below... see DESIGN.md): caller takes its own path    */
    LGW_BODY_ENCODE_ERROR = 5   /* the reference's encoder raises (NaN/Infinity under allow_nan=False, lone surrogate under
                                   ensure_ascii=False): the attempt fails at request_handler.py:183                            */
};
typedef struct lgw_body_op {        /* one `payload[key] = value` */
    uint32_t key_off, key_len;      /* key text (UTF-8) in the blob */
    uint32_t rkey_off, rkey_len;    /* key as the mode renders it   */
    uint32_t rval_off, rval_len;    /* value as the mode renders it */
    uint32_t flags;                 /* bit0: only when the client's body lacks the key (chat.py:114)
                                       bit1: presence probe: nothing assigned/appended, only reported in lgw_body_result.matched */
    uint32_t _pad;
} lgw_body_op;
#define LGW_PLAN_RESPONSE 0x100u     /* or-ed into lgw_body_plan.mode: the document is an upstream RESPONSE (row a12) */
typedef struct lgw_body_plan { uint32_t op_begin, op_end, mode, _pad; } lgw_body_plan;
typedef struct lgw_body_result {
    uint32_t status, out_len;
    uint32_t matched;               /* bit i: op i's key is present at the top level of the body (response plans on a root
                                       that is not an object: Python's `in` -- an element of the list equals the key, the key is a
                                       substring of the string) */
    uint32_t root_kind;             /* lgw_kind of the document's root value */
} lgw_body_result;
typedef struct lgw_body_scan {
    uint32_t status;                /* LGW_BODY_OK / PARSE_ERROR / NO_MODEL */
    uint32_t model_len;             /* bytes of the model string (may exceed model_cap: truncated) */
    uint8_t model_kind, model_truthy, stream_kind, stream_truthy;   /* lgw_kind of body["model"], body.get("stream") */
    uint32_t _pad;
} lgw_body_scan;

/* upload the compiled plan table (replaces the previous one; at most 32 ops per plan) */
int lgw_rules_load(lgw_engine* e, const lgw_body_plan* plans, uint32_t n_plans,
                   const lgw_body_op* ops, uint32_t n_ops, const uint8_t* blob, uint32_t blob_len);
/* chat.py:31-45 for n bodies: host pointers; models_out = n slots of model_cap bytes */
int lgw_bodies_scan(lgw_engine* e, const uint8_t* bodies, const uint64_t* body_off /* n+1 */, uint32_t n,
                    uint32_t model_cap, lgw_body_scan* scans_out, uint8_t* models_out);
/* one attempt's payload bytes for n bodies: body i is rewritten by plan plan_idx[i].  Outputs are packed
 * back to back: body i occupies out[out_off[i] .. out_off[i+1]) (empty unless status OK).  out_cap is the
 * size of `out`; slot_cap bounds one output (bodies needing more report LGW_BODY_OVERFLOW). */
int lgw_bodies_rewrite(lgw_engine* e, const uint8_t* bodies, const uint64_t* body_off /* n+1 */, uint32_t n,
                       const uint32_t* plan_idx, uint32_t slot_cap,
                       uint8_t* out, uint64_t out_cap, uint64_t* out_off /* n+1 */, lgw_body_result* results);
/* same with every pointer in device memory (bench `value`, callers that keep bodies resident) */
int lgw_bodies_rewrite_device(lgw_engine* e, const uint8_t* d_bodies, const uint64_t* d_body_off, uint32_t n,
                              uint64_t n_bytes, const uint32_t* d_plan_idx, uint32_t slot_cap,
                              uint8_t* d_out, uint64_t out_cap, uint64_t* d_out_off, lgw_body_result* d_results);
/* device time of the last rewrite's kernels (rewrite, offsets, pack), milliseconds */
int lgw_bodies_last_ms(lgw_engine* e, float ms[3]);

/* ---- response tap of NON-streaming responses: SURVEY 8 row a8, chat_logging.py:98-103,:113-150 -------------------------------
 * The tap thread concatenates the chunks of a non-event-stream response and treats the whole text as ONE part (:105-106): it must
 * start with `{` (or `data: {`), is parsed once (:123), walks `choices` (:124-133), takes get_token_usage of the document when it
 * has a "usage" key (:134-135), writes an extra row when it has an "error" key (:137-139) and the final row (:150).  One result per
 * document: the record of that final row (the defaults when nothing was taken) and what else happened. */
typedef struct lgw_doc_usage {
    uint32_t flags;              /* TopKey | PartFlag bits of the parse (0: the text was not taken as JSON) */
    uint8_t rec_valid;           /* 1: rec = get_token_usage(document); 0: rec = the defaults of chat_logging.py:77-84 */
    uint8_t error_row;           /* 1: the document has a top-level "error": the same record is written once more before the final row */
    uint8_t exotic;              /* 1: a shape the device does not model (reported, never guessed) */
    uint8_t _pad;
    lgw_usage_rec rec;
} lgw_doc_usage;
/* host pointers; document i is docs[doc_off[i] .. doc_off[i+1]) */
int lgw_documents_usage(lgw_engine* e, const uint8_t* docs, const uint64_t* doc_off /* n+1 */, uint32_t n, lgw_doc_usage* out);

/* ---- error detail of a failing non-streaming upstream response (SURVEY.md row a12; request_handler.py:167-169) ----
 *     error_detail = response_json.get("error", {}).get("message") or response_json.get("detail")
 * for documents that lgw_bodies_rewrite (response plan) reported as valid JSON with an object root and a top-level "error" or
 * "detail" key.  result: 0 None, 1 a str (text[i*text_stride ..][0..text_len), UTF-8, unescaped), 2 True, 3 False,
 * 4 "error" is not an object (`.get` raises AttributeError: the type name follows from error_kind; for a number the text holds
 * its literal), 5 not modelled (a non-empty container wins, a lone surrogate, text longer than text_stride), 6 a number wins:
 * the text holds its literal as spelt in the document.  kinds: 0 absent, 1 string, 2 null, 3 true, 4 false, 5 numeric zero, 6 number, 7 {}, 8 object, 9 [], 10 array. */
typedef struct lgw_doc_error {
    uint8_t result;
    uint8_t error_kind, message_kind, detail_kind;
    uint32_t text_len;
} lgw_doc_error;
int lgw_documents_error_detail(lgw_engine* e, const uint8_t* docs, const uint64_t* doc_off /* n+1 */, uint32_t n, lgw_doc_error* out,
                               uint8_t* text, uint32_t text_stride);

/* ---- transcript tap: SURVEY 8(f) rank 3, chat_logging.py:108-139 -------------------------------------------------------------------
 * The other half of the response tap: the text ChunkProcessorThread accumulates in `llm_response_accum` -- for every parsed event, for
 * every choice, `delta.content` else `message.content` when truthy (:124-133), JSON escapes decoded; a top-level "error" appends the
 * event's own stripped text and calls write_log at once with the text so far (:137-139).  Optional, like the reference's tap
 * (LOG_CHAT_ENABLED, :166-168): lgw_transcripts_enable allocates the per-stream tap state; streams opened afterwards are tapped.
 *
 * After each lgw_sse_step / lgw_sse_step_device (and before the next one) lgw_step_transcript_run walks the chunks that step RELAYED
 * (seg_out[s].emit_chunk_begin onward) with the tap's own carry and leaves on the device: the text appended per segment, packed
 * segment after segment (UTF-8; a lone surrogate escape is written in 'surrogatepass' form and flagged), and the marks -- mid-stream
 * write_log calls: the transcript written at mark (slot, seq) is the stream's text up to byte text_pos (counted from the stream's
 * start).  It returns the sizes; lgw_step_transcript_fetch copies them out: text_out[seg_text_off[s] .. seg_text_off[s+1]) is what
 * segment s appended.  File naming, the header block and log pruning of write_log (:22-67) stay on the host
 * (llmapigateway_b200/transcripts.py). */
enum lgw_text_flag {
    LGW_TF_LONE_SURROGATE = 1 << 0,  /* the stream's text holds a lone surrogate: the reference's f.write raises (no file, no DB row) */
    LGW_TF_EXOTIC = 1 << 1,          /* an event shape whose Python behaviour the device does not model: text not authoritative */
    LGW_TF_CARRY_OVERFLOW = 1 << 2,  /* an unterminated event outgrew carry_cap */
    LGW_TF_MARKQ_OVERFLOW = 1 << 3,  /* more marks in one step than rowq_cap */
    LGW_TF_SEQUENTIAL = 1 << 4,      /* (this step) the segment took the sequential walk */
    LGW_TF_DOC_ERROR_LOG = 1 << 5    /* (lgw_documents_text) the document has a top-level "error": write_log ran at :139 too */
};
typedef struct lgw_text_mark { uint32_t slot, seq; uint64_t text_pos; } lgw_text_mark;
int lgw_transcripts_enable(lgw_engine* e);
int lgw_step_transcript_run(lgw_engine* e, uint64_t* text_bytes, uint32_t* n_marks);
int lgw_step_transcript_fetch(lgw_engine* e, uint8_t* text_out /* text_bytes */, uint64_t* seg_text_off /* n_segs+1 */,
                              uint32_t* seg_flags /* n_segs */, lgw_text_mark* marks_out /* n_marks */);
/* device time of the last transcript pass (extract + scan + pack), milliseconds */
int lgw_transcript_last_ms(lgw_engine* e, float* ms);

/* text the non-streaming tap accumulates for each document (chat_logging.py:97-150, the documents of lgw_documents_usage): the whole
 * document is one part; for every choice `delta.content` else `message.content` when truthy, JSON escapes decoded, plus the document's
 * own text when it has a top-level "error".  Text of doc i = text_out[text_off[i] .. text_off[i+1]) (UTF-8, a lone surrogate in
 * 'surrogatepass' form); flags[i]: LGW_TF_LONE_SURROGATE / LGW_TF_EXOTIC, and LGW_TF_DOC_ERROR_LOG when write_log ran at :139 as
 * well as at :150 (both calls write this text).  A text_cap of twice the batch's bytes always suffices; when the text does not fit
 * the call returns LGW_ERR_CAPACITY before anything is copied out.  Documents are limited to 2^31 bytes. */
int lgw_documents_text(lgw_engine* e, const uint8_t* docs, const uint64_t* doc_off /* n+1 */, uint32_t n,
                       uint8_t* text_out, uint64_t text_cap, uint64_t* text_off /* n+1 */, uint32_t* flags /* n */);
/* device time of the last lgw_documents_text (walk + scan + pack), milliseconds */
int lgw_documents_text_last_ms(lgw_engine* e, float* ms);

/* ---- device memory helpers for callers without their own CUDA allocator ----------------------------- */
int lgw_device_alloc(lgw_engine* e, uint64_t bytes, void** out);
int lgw_device_free(lgw_engine* e, void* p);
int lgw_device_upload(lgw_engine* e, void* d_dst, const void* h_src, uint64_t bytes);
int lgw_device_download(lgw_engine* e, void* h_dst, const void* d_src, uint64_t bytes);
int lgw_device_zero(lgw_engine* e, void* d_dst, uint64_t bytes);

/* ---- pinned staging buffers (SURVEY 8(b) ownership) -------------------------------------------- */
int lgw_alloc_pinned(lgw_engine* e, uint64_t bytes, void** out);
int lgw_free_pinned(lgw_engine* e, void* p);

#ifdef __cplusplus
}
#endif
#endif /* LLMGW_B200_H */
