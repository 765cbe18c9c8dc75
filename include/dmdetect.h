/*
 * dmdetect.h -- C ABI of libdmdetect.so, the H100 (sm_90a) detector hot path.
 *
 * The reference has no FFI: its hot path is the Python call chain
 *   Engine._run_loop            /root/reference/src/service/features/engine.py:153-217
 *     -> Service.process        /root/reference/src/service/core.py:176-206
 *       -> CoreComponent.process (detectmatelibrary, un-vendored; contract in
 *                                 /root/reference/docs/interfaces.md:23-35)
 * This header is what a `process(bytes) -> bytes | None` implementation binds instead of
 * the library's Python detector; INTEGRATION.md shows the ctypes stub.  Plain pointers and
 * sizes only -- no torch / CUDA runtime types cross the boundary (a CUDA stream is passed
 * as an opaque void*, NULL = the handle's own stream).
 *
 * Conventions
 *   - every entry point returns 0 on success or a negative DM_ERR_* code; the message of
 *     the last failure on the calling thread is dm_last_error().  Nothing throws.
 *   - one handle = one device = one caller thread at a time (the reference calls process()
 *     from the single EngineLoop thread only, engine.py:80-82).
 *   - the caller owns every buffer it passes in; the library owns its tables and scratch
 *     (allocated in dm_create or on first use, and grown when a batch needs more;
 *     dm_import_known stages the keys it is given in a buffer of its own).
 *   - there is NO CPU fallback: without a usable CUDA device dm_create fails.
 */
#ifndef DMDETECT_H
#define DMDETECT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DM_ABI_VERSION 4
#define DM_MAX_KEYS 32      /* monitored fields per detector                         */
#define DM_MAX_KEYLEN 32    /* bytes per monitored key                                */

#define DM_OK 0
#define DM_ERR_ARG (-1)       /* bad argument                                         */
#define DM_ERR_CUDA (-2)      /* CUDA runtime / launch failure (see dm_last_error)    */
#define DM_ERR_NO_DEVICE (-3) /* no usable sm_90 device: the product has no CPU path */
#define DM_ERR_CAPACITY (-4)  /* batch larger than the handle was created for         */
#define DM_ERR_TABLE_FULL (-5)/* known-set table over its load limit                  */
#define DM_ERR_STATE (-6)     /* call not valid in the handle's current state         */

typedef struct dm_handle dm_handle;

/* Running statistics of one handle (the "per-window running statistics" that are
 * all-reduced across GPUs; replaces the Python-side counters the reference keeps in
 * core.py:24-61 for lines/bytes, plus what NewValueDetector reports per alert). */
typedef struct {
    uint64_t lines;          /* records seen (training + detection)                   */
    uint64_t train_lines;    /* records consumed as training data                     */
    uint64_t detect_lines;   /* records scored                                        */
    uint64_t anomalies;      /* records with score > 0                                */
    uint64_t score_sum;      /* sum of scores (scores are small integers)             */
    uint64_t bytes;          /* input bytes consumed                                  */
    uint64_t known_keys;     /* entries in the known-set table                        */
    uint64_t bad_records;    /* records that could not be parsed (malformed ParserSchema,
                                see dm_process_records; log_format mismatch): counted,
                                never trained or scored                               */
    uint64_t unknown_per_key[DM_MAX_KEYS]; /* alerts per monitored field             */
} dm_stats_t;

/* One anomalous record of the last batch. */
typedef struct {
    uint32_t line;    /* record index inside the batch                                */
    uint32_t mask;    /* bit k set = monitored field k held an unknown value          */
    uint64_t offset;  /* byte offset of the record's first byte inside the batch      */
} dm_anomaly_t;

const char* dm_last_error(void);
int dm_abi_version(void);

/* Create a detector on CUDA device `device`.
 *   keys_blob/key_lens : the n_keys monitored field names, concatenated (R-tok keys:
 *                        1..DM_MAX_KEYLEN bytes, none of ' ', '"', '\'', '=', '\n').
 *                        Field k is the reference's monitor k
 *                        (container/config/detector_config.yaml:6-9, header_variables pos).
 *   max_batch_bytes    : largest message dm_process_lines will be given.
 *   max_lines          : largest record count per message (0 = max_batch_bytes / 8).
 *   table_log2_slots   : known-set table capacity = 2^table_log2_slots keys (10..28). */
int dm_create(int device, uint32_t n_keys, const uint8_t* keys_blob, const uint32_t* key_lens,
              uint64_t max_batch_bytes, uint64_t max_lines, uint32_t table_log2_slots,
              dm_handle** out);
int dm_destroy(dm_handle* h);

/* The hot path: one message of '\n'-terminated raw records (R-tok L1).
 *   buf, nbytes      : the message; host memory (pageable or pinned) or, if buf_on_device,
 *                      a 16-byte aligned device pointer with >= 16 readable bytes of slack
 *                      after nbytes.
 *   n_train_lines    : the first n_train_lines records of THIS message are training data
 *                      (R-spec 1): their values are inserted, their flag/score are 0.  The
 *                      rest are scored against the table as it stands after that insert.
 *   flags_out/scores_out : one uint8 flag and one float32 score per record, capacity
 *                      out_cap_lines; host memory, or device memory if out_on_device.
 *                      Either may be NULL (results then stay in the handle's own buffers).
 *   n_lines_out/n_anomalies_out : host pointers, may be NULL.  If both are NULL and no host
 *                      output was requested the call only ENQUEUES work on `stream` and
 *                      returns without synchronising (device-resident pipelines; its errors are reported by
 *                      the next dm_sync or synchronous call); otherwise it returns after the results are
 *                      complete.
 * Call order: a handle's calls take effect in the order they are made, whatever stream each one uses (`stream` here,
 * the handle's own stream for the other entry points).  A call on another stream than the handle's previous call
 * first waits, on the device, for that stream, so it sees the known-set table, statistics and errors of every earlier
 * call; calls that stay on one stream add no waits.  Two kinds of call keep the ordering documented with them: the
 * window calls (dm_window_export / _import / _allreduce), which the caller orders, so that two all-reduces can be in
 * flight; and dm_encode_alerts of a collected slot, which is ordered behind that slot only, so that the other slot
 * stays in flight.
 * By default a call is ordered behind everything enqueued on `stream` before it.  After
 * dm_set_overlap(h, 1) consecutive device-resident detection calls on one stream overlap
 * (programmatic dependent launch): a call may then start READING its `buf` and the known-set
 * table while the previous call's kernel is still running (outputs, header and statistics are
 * still written in call order).  That is only safe when the caller does not enqueue, between
 * two calls on that stream, a KERNEL that writes the next call's `buf` -- copies (cudaMemcpyAsync)
 * and event waits are fine, they are ordered in full.  dm_submit_lines always overlaps (its
 * inputs arrive by copy).
 * Replaces: per-record CoreComponent.process calls made by core.py:201-203. */
int dm_process_lines(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int buf_on_device,
                     uint64_t n_train_lines,
                     uint8_t* flags_out, float* scores_out, uint64_t out_cap_lines, int out_on_device,
                     uint64_t* n_lines_out, uint64_t* n_anomalies_out, void* stream);

/* Switch the overlap of consecutive dm_process_lines calls (see above) on or off; off at creation
 * (DM_OVERLAP=1 in the environment turns it on for every handle). */
int dm_set_overlap(dm_handle* h, int on);

/* Record mode: the detector fed with already-extracted values, as when the upstream parser
 * sends one ParserSchema per message (engine.py:163-187; the host decodes the protobuf
 * framing, docs/interfaces.md:124-128).  Value i is blob[offsets[i], offsets[i+1]) and
 * belongs to monitored field fields[i] of record record_of[i].  Records
 * [0, n_train_records) are training data; the rest are scored: flags_out / scores_out /
 * masks_out have n_records entries (host memory, any may be NULL).  Synchronous. */
int dm_process_values(dm_handle* h, const uint8_t* blob, uint64_t blob_bytes, const uint32_t* offsets,
                      const uint32_t* fields, const uint32_t* record_of, uint32_t n_values,
                      uint32_t n_records, uint32_t n_train_records, uint64_t record_bytes,
                      uint8_t* flags_out, float* scores_out, uint32_t* masks_out,
                      uint64_t* n_anomalies_out);

/* Record mode on the device: a message holding a BATCH of serialized ParserSchema records,
 * each preceded by its varint length (protobuf "delimited" framing; a message that holds a
 * single bare record is the reference's native case and goes through dm_process_values).
 * The host only walks the length prefixes; the protobuf field walk, the monitor matching
 * (dm_set_monitors), dm_fp64, the table probe and the scoring run in one kernel, one thread
 * per record.  Host output buffers of out_cap entries (any may be NULL).  Synchronous.
 * Replaces per-record ParserSchema.deserialize + NewValueDetector.train/detect behind
 * core.py:201-203.
 * A record is well-formed if and only if protobuf's runtime parses it as ParserSchema
 * (strict UTF-8 in every string field and map key / value, tags below 2^32 and not field 0,
 * every payload inside the record), with one deliberate exception: a record holding a group
 * (wire types 3/4) is malformed, where protobuf skips it (proto3 cannot declare groups).  A
 * well-formed record yields the values protobuf yields; a map entry holding any field but
 * LEN fields 1 and 2 is dropped, as protobuf drops it.  A malformed record gets flag, score
 * and mask 0, is counted in dm_stats_t.bad_records and is never trained on.
 * Training: the first n_train_records WELL-FORMED records train (malformed records take no
 * training slot); every record from just past the n_train_records-th well-formed one is
 * scored.  dm_stats_t.train_lines grows by the records trained; the bad_records delta of a
 * call is the number of its malformed records. */
typedef struct {
    int32_t event_id;     /* records with this EventID only ...                          */
    uint32_t has_event;   /* ... if non-zero; 0 = global scope (every record)            */
    uint32_t source;      /* 0 = header variable logFormatVariables[key], 1 = variables[var_index] */
    uint32_t var_index;
    uint32_t key_len;
    uint8_t key[64];
} dm_monitor_t;
int dm_set_monitors(dm_handle* h, uint32_t n_monitors, const dm_monitor_t* monitors);
/* Combination monitors -- NewValueComboDetector (named at
 * src/service/features/component_resolver.py:15,39-40; config shape
 * tests/test_reconfigure_params.py:149-169): combination c is the ordered tuple of the
 * values of monitors members[member_off[c] .. member_off[c+1]); a record yields it when all
 * of them are present (and in scope).  It is learnt / looked up in the same table under
 * field n_monitors + c and reported in bit n_monitors + c of the masks of
 * dm_process_records (n_monitors + n_combos <= 32).  Monitors whose bit is set in
 * member_only_mask do not alert on their own.  Call after dm_set_monitors (which clears the
 * combinations).  Applies to dm_process_records, to dm_process_lines on key=value records
 * (monitor k = field k of dm_create; the library then uses its one-thread-per-record kernel,
 * dm_get_anomalies reports the same mask bits) and to dm_process_lines in log_format mode
 * (dm_set_format[_ex], before or after this call): a member is present when the same monitor
 * would be scored on its own -- the log_format matched, the record is in scope, the capture
 * exists / the variable index is below the matched template's wildcard count; an empty
 * capture is present.  Under R-norm a variable member's value is its slice of the normalised
 * Content.  The key of a tuple is the same in all three modes.  Not the pipelined path. */
int dm_set_combos(dm_handle* h, uint32_t n_combos, const uint32_t* member_off, const uint32_t* members,
                  uint32_t member_only_mask);
/* MatcherParser fused in front of the detector (SURVEY.md section 8f-3).  Replaces
 * detectmatelibrary.parsers.template_matcher.MatcherParser as configured at
 * tests/library_integration/test_pipe_filereader_matcher_nvd.py:74-88 and
 * docs/getting_started.md:395-415, i.e. the parser service upstream of core.py:201-203.
 *   log_format   literal text with <Name> captures, e.g.
 *                `<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"`
 *                or `type=<type> msg=audit(<Time>): <Content>`; captures are the record's header
 *                variables (logFormatVariables).  Semantics = ^L0(.*?)L1(.*?)...$ with escaped
 *                literals (non-greedy captures, last one to the end).
 *   templates    `<*>` wildcard templates matched in order against the capture named
 *                content_name (NULL = "Content"); the first match sets EventID = its index
 *                (0-based, -1 = no match) and variables[i] = its i-th wildcard.
 * The monitors of dm_set_monitors are bound to it: header monitors by capture name, variable
 * monitors by wildcard index, event scope by EventID.  After this call dm_process_lines
 * tokenises with the log_format instead of key=value fields (one thread per record); records
 * the log_format does not match are counted (dm_stats_t.bad_records) and never alert.
 * log_format = NULL switches back.  Limits (DM_ERR_ARG): at most 63 templates and 32 captures
 * per chain; every literal at most 255 bytes (template literals after R-norm); at most 512
 * literals and 4096 bytes of literal text over the log_format and all templates, each literal
 * counted rounded up to whole 4-byte words.  The strings end at their first NUL byte. */
int dm_set_format(dm_handle* h, const char* log_format, const char* content_name, uint32_t n_templates,
                  const char* const* templates);
/* dm_set_format + MatcherParser's params.remove_spaces / remove_punctuation / lowercase
 * (tests/library_integration/test_pipe_filereader_matcher_nvd.py:82-84 sets all three).
 * norm_flags = OR of DM_NORM_*: before template matching the Content text and the literal
 * parts of every template (the `<*>` stay) lose ASCII white space (0x09-0x0D, 0x20) and/or the
 * 32 ASCII punctuation bytes, and/or have 'A'-'Z' folded to lower case; variables[i] are then
 * slices of the normalised Content.  Header captures are never normalised.  (DESIGN.md R-norm;
 * the library is not vendored in the reference, so this rule is unpinned.) */
#define DM_NORM_REMOVE_SPACES 1u
#define DM_NORM_REMOVE_PUNCTUATION 2u
#define DM_NORM_LOWERCASE 4u
int dm_set_format_ex(dm_handle* h, const char* log_format, const char* content_name, uint32_t n_templates,
                     const char* const* templates, uint32_t norm_flags);
/* Diagnostics: 1 if the last key=value message was processed by the stream kernel's batch-wise re-check of candidate
 * fields, 0 if candidates were re-checked one by one.  Both give the same results; unless DM_STREAM_RECHECK=thread|chain
 * pins it, the library chooses per message from how often the previous message's field batches held a candidate. */
int dm_stream_recheck_chained(dm_handle* h);
/* Host utility: write a host buffer back to memory and evict it from the CPU caches (x86:
 * clflush), so that device DMA streams it from DRAM instead of snooping dirty cache lines. */
int dm_host_cache_flush(const void* p, uint64_t nbytes);

/* Diagnostics: {smid, t_start, t_rows_done, t_exit} (globaltimer ns) of every CTA of the last stream-kernel
 * launch, followed by 8 time stamps of its epilogue; *n_warps_out = number of CTAs.  Only for handles created
 * with DM_STREAM_TIMELINE=1 in the environment (scripts/stream_timeline.py).  The name is historical. */
int dm_debug_rows_timeline(dm_handle* h, unsigned long long* out, uint64_t cap_words, uint32_t* n_warps_out);
int dm_process_records(dm_handle* h, const uint8_t* buf, uint64_t nbytes, uint32_t n_train_records,
                       uint8_t* flags_out, float* scores_out, uint32_t* masks_out, uint64_t out_cap,
                       uint64_t* n_records_out, uint64_t* n_anomalies_out);

/* LogSchema input: what the reader stage sends (one serialized LogSchema per message), so that the detector -- with
 * dm_set_format[_ex] the parser and the detector fused -- can stand where the parser service stands.
 *   delimited = 0: buf is ONE bare LogSchema record; 1: varint-length-delimited records.
 * Each record's text is unwrapped on the device and the texts go through dm_process_lines' detection unchanged
 * (key=value or log_format mode, combinations included).  Rule R-log (DESIGN.md):
 *   - a record is well-formed if and only if protobuf's runtime parses it as LogSchema (fields 1-5 are strings, strict
 *     UTF-8 in all of them), with the same exception as dm_process_records: a group makes it malformed;
 *   - its text is its `log` field (the last one wins; absent = "") less ONE trailing '\n'; a text that still holds a
 *     '\n' is unusable;
 *   - malformed and unusable records get flag and score 0, count in dm_stats_t.bad_records and take no training slot;
 *   - every other record gets exactly the result its text gets as a line of a dm_process_lines message made of the
 *     usable texts, each followed by '\n', in order; the first n_train_records of them train.
 * flags_out / scores_out: host buffers of out_cap entries, one per record (either may be NULL).  *n_malformed_out =
 * malformed + unusable records.  dm_get_anomalies then reports (record index, mask, byte offset of the record's payload
 * in buf).  Statistics: lines += records, bytes += nbytes, train_lines / detect_lines as dm_process_records counts them.
 * Synchronous; ends the overlap chain of dm_process_lines (dm_set_overlap).  Not the pipelined path. */
int dm_process_logs(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int delimited, uint32_t n_train_records,
                    uint8_t* flags_out, float* scores_out, uint64_t out_cap,
                    uint64_t* n_records_out, uint64_t* n_malformed_out, uint64_t* n_anomalies_out);

/* DetectorSchema alerts of the last batch, encoded on the device (rule R-alert, DESIGN.md): the bytes the component's
 * host encoder writes for the same batch (component.py _process_lines_one / _process_logs / _process_record_batch,
 * _detector_schema, wire.encode_detector_schema), for raw lines and LogSchema records in key=value mode and in
 * log_format mode (dm_set_format[_ex]), and for ParserSchema records.
 * dm_set_alert_format fixes what does not change from call to call and allocates, once, the device buffers, of which
 * the output buffer holds out_cap bytes:
 *   strings / string_lens : n_strings strings, concatenated: __version__, detectorID, detectorType, description, then
 *                           the alert keys (alertsObtain keys) in output order, i.e. sorted by their UTF-8 bytes;
 *   bits_off / bits       : alert key j is supplied by the mask bits bits[bits_off[j], bits_off[j + 1]) in config
 *                           order; of those set in a record's mask the last one wins.  A bit below n_keys is monitor
 *                           k, worded "Unknown value: '<v>'"; bit n_keys + c is combination c, whose monitors are
 *                           combo_members[combo_off[c], combo_off[c + 1]) ("Unknown value combination: ('<v1>', ...)").
 *                           Monitor k's value: key=value mode, the first true field of key k of dm_create (R-tok
 *                           L2-L6); log_format mode, its header capture verbatim or its template variable (under
 *                           R-norm a slice of the normalised Content); ParserSchema records, the value the
 *                           monitor of dm_set_monitors reads (logFormatVariables[key], last entry wins, or
 *                           variables[i]);
 *   time_capture          : log_format mode: the header capture whose text is the record's Time, 0xFFFFFFFF = none
 *                           (key=value mode always takes msg=audit(<Time>...), R-tok L7).
 * dm_encode_alerts encodes the last batch of dm_process_lines (whichever kernel ran it), dm_process_logs,
 * dm_process_records or dm_collect (a slot of the pipelined path, worded as a dm_process_lines batch) into `out`: one
 * varint-length-delimited DetectorSchema per anomalous record, in record order;
 * alertID = first_alert_id + j (signed), detectionTimestamp = receivedTimestamp = now, extractedTimestamps =
 * [int(float(Time))], or now when the record has no Time or its Time is no float literal.  logIDs = [first_log_id +
 * record index] for raw lines; the record's own logID (LogSchema field 2, ParserSchema field 8, the last one; "" when
 * absent) for the other two, which ignore first_log_id.  Time: raw lines and LogSchema texts as R-alert reads them;
 * ParserSchema, logFormatVariables["Time"] (absent = now).  *n_alerts = anomalous records, *out_len = bytes.
 * *declined = 1 when the device cannot give the host's bytes: a Time string it cannot convert with certainty (outside
 * [0-9]{1,10}(\.[0-9]{0,6})? yet made only of bytes a float literal may hold; for ParserSchema also any Time holding a
 * byte >= 0x80 and no ASCII byte a float literal cannot hold), a ParserSchema batch with more anomalous records than
 * the anomaly list holds (*out_len is then 0), or an output larger than min(out_cap, the out_cap of
 * dm_set_alert_format) (*out_len then tells how large); the caller then encodes that batch on the host.
 * Synchronous; ends the overlap chain of dm_process_lines.  The encoder reads the batch's message, its scores and its
 * anomaly list, which the next overlapped call rewrites; so a device-resident caller must leave that call's `buf` --
 * and its `scores_out`, when it passed a device scores buffer -- unchanged until dm_encode_alerts returns, and must not
 * enqueue another dm_process_lines on the handle in between.  A collected slot is encoded on a stream that follows its
 * kernels, while the other slot's message stays in flight; the slot's input and anomaly list must survive until the
 * call returns, so call it after dm_collect(slot) and before the next dm_submit_lines on that slot (with two slots in
 * turn: collect piece i, encode it, then submit piece i + 2).  DM_ERR_STATE when the last batch came from another
 * entry point (dm_process_values, dm_parse_logs, dm_import_known) or dm_submit_lines was called since. */
int dm_set_alert_format(dm_handle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* string_lens,
                        const uint32_t* bits_off, const uint32_t* bits, uint32_t n_combos, const uint32_t* combo_off,
                        const uint32_t* combo_members, uint32_t time_capture, uint64_t out_cap);
int dm_encode_alerts(dm_handle* h, uint64_t first_log_id, int64_t first_alert_id, int64_t now, uint8_t* out,
                     uint64_t out_cap, uint64_t* out_len, uint64_t* n_alerts, int* declined);

/* The MatcherParser stage on the device (rule R-parse, DESIGN.md): LogSchema records in, ParserSchema records out,
 * the bytes the parser component's host path writes (parser.py, wire.encode_parser_schema).  The detector's known set
 * is not touched: a handle with n_keys = 0 (dm_set_monitors with no monitors) and the smallest table is enough.
 * dm_set_parser_format, after dm_set_format[_ex] (and again after every later dm_set_format[_ex]): n_strings strings,
 * concatenated: __version__, parserType, parserID, the template texts verbatim in EventID order, then the names of the
 * log_format's captures in output order (sorted by their UTF-8 bytes); name j is capture capture_order[j].
 * dm_parse_logs takes one bare LogSchema record (delimited = 0) or a varint-length-delimited batch, framed and checked
 * as dm_process_logs (R-log).  A malformed or unusable record gives no output; every other one gives one ParserSchema:
 *   EventID    the template the Content matched (-1: none, or the log_format did not match)
 *   template   that template's text (EventID >= 0 only); variables: its wildcards (slices of the R-norm Content)
 *   parsedLogID  first_parsed_id + the number of records emitted before it in this call, in decimal
 *   logID      the record's last field 2 ("" when absent); log: its text
 *   logFormatVariables  every capture of the log_format, when it matched
 *   receivedTimestamp = parsedTimestamp = now
 * *out = the varint-length-delimited ParserSchemas in record order, *out_len bytes, in a pinned buffer the handle owns,
 * valid until the next dm_parse_logs.  *n_emitted = ParserSchemas, *n_malformed = malformed + unusable records.
 * Synchronous; ends the overlap chain of dm_process_lines, and dm_encode_alerts no longer has a batch to encode. */
int dm_set_parser_format(dm_handle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* string_lens,
                         const uint32_t* capture_order);
int dm_parse_logs(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int delimited, int64_t first_parsed_id, int64_t now,
                  const uint8_t** out, uint64_t* out_len, uint64_t* n_records_out, uint64_t* n_emitted_out,
                  uint64_t* n_malformed_out);

/* Pipelined host path (two slots): dm_submit_lines enqueues, without waiting, the copy of a
 * HOST message (pinned memory gives real overlap) to the device, the kernels and the copy
 * of the batch header back; dm_collect waits for that slot, copies the slot's flags and
 * scores into pinned buffers owned by the handle and returns pointers to them (valid until
 * the slot is submitted again).  While slot 1's message is crossing PCIe, slot 0's kernels
 * run and its results travel back.  Messages are processed in submission order (training
 * before detection is preserved).  Raw-mode equivalent of calling dm_process_lines per
 * message; replaces the same per-record calls of core.py:201-203.  dm_submit_lines leaves the
 * handle without a last batch; dm_collect makes the slot's batch the last batch, which
 * dm_encode_alerts can then word (see there for how long the slot must stay untouched). */
int dm_submit_lines(dm_handle* h, const uint8_t* host_buf, uint64_t nbytes, uint64_t n_train_lines, uint32_t slot);
int dm_collect(dm_handle* h, uint32_t slot, const uint8_t** flags_out, const float** scores_out,
               uint64_t* n_lines_out, uint64_t* n_anomalies_out);
/* Anomalous records of the batch last collected from `slot` (same format as dm_get_anomalies). */
int dm_collect_anomalies(dm_handle* h, uint32_t slot, dm_anomaly_t* out, uint32_t cap, uint32_t* n_out);

/* Wait for everything enqueued on the handle, whatever streams it went to (see "Call order" at dm_process_lines; of the
 * window calls, the last dm_window_import), and report the last batch's counts.  On the default key=value kernel
 * the error reported is that of ANY dm_process_lines call since the last dm_sync or synchronous dm_process_lines (a
 * message with more records than out_cap_lines or max_lines, a training message that filled the known-set table, an
 * anomaly list that overflowed), not only of the last one: an enqueued message whose outputs are wrong or truncated
 * is not hidden by a good message behind it.  Reporting them clears them.  (DM_KERNEL=lanes, log_format mode and
 * combination monitors report the last call's errors only.) */
int dm_sync(dm_handle* h, uint64_t* n_lines_out, uint64_t* n_anomalies_out);

/* The anomalous records of the last batch, sorted by record index (at most cap; *n_out is
 * the total found, which may exceed cap and the handle's internal list). */
int dm_get_anomalies(dm_handle* h, dm_anomaly_t* out, uint32_t cap, uint32_t* n_out);

int dm_get_stats(dm_handle* h, dm_stats_t* out);

/* Known-set persistence (the reference loses learned state on restart, SURVEY.md 5).
 * dm_export_known: every key of the table, strictly ascending; *n_out = their count, at most cap copied to keys_out
 * (host memory).  Compaction and sort run on the device; cap 0 (or keys_out NULL) only reads the count.  The first
 * export that copies keys allocates a device scratch of two slots/2-key buffers, kept until dm_destroy. */
int dm_export_known(dm_handle* h, uint64_t* keys_out, uint64_t cap, uint64_t* n_out);
int dm_import_known(dm_handle* h, const uint64_t* keys, uint64_t n);
/* Forget everything learned and zero the statistics. */
int dm_reset(dm_handle* h);

/* Host-side helper: table key of (field k, value) = dm_fp64(value) ^ salt(k).  Pure
 * function, no device needed -- lets a host seed/inspect the known set by value. */
uint64_t dm_table_key(uint32_t field, const uint8_t* value, uint32_t len);

/* Multi-GPU window exchange: ONE sum-all-reduce of `dm_window_words(world)` uint64 words
 * per window carries the statistics delta and every rank's newly learned keys
 * (rank r writes its keys only into segment r, so the sum is a concatenation).
 *   export : pack this rank's delta since the previous window into dev_buf (device memory).
 *   (caller all-reduces dev_buf with SUM over uint64 -- NCCL over NVLink via torch.distributed)
 *   import : insert all ranks' keys into the local table, fold the global statistics.
 * Export and import run on `stream` (NULL: the handle's own).  An import with keys changes the table that detection
 * reads: the caller orders it before any later detection on the handle (e.g. the same stream).  An import's errors
 * (the table over its load limit) are reported by the next dm_sync or synchronous dm_process_lines. */
uint64_t dm_window_words(dm_handle* h, uint32_t world, int with_keys);
int dm_window_export(dm_handle* h, uint64_t* dev_buf, uint32_t rank, uint32_t world, int with_keys, void* stream);
int dm_window_import(dm_handle* h, const uint64_t* dev_buf, uint32_t rank, uint32_t world, int with_keys, void* stream);
/* A window carries at most 65536 newly learnt keys per rank.  After an export with keys: how many of this rank's
 * learnt keys are still waiting (0 in all but pathological training windows).  When any rank reports > 0 the caller
 * runs another exchange with keys before detection starts (all ranks call the collective the same number of times);
 * window.DeviceWindow.exchange does so.  dm_window_allreduce's export sets the count too. */
int dm_window_pending_keys(dm_handle* h, uint64_t* n_out);

/* The same exchange done by the library itself: export, ncclAllReduce(sum, uint64) over the
 * handle's own communicator, import -- enqueued on `stream` by ONE call (no host work per
 * window besides this call).  NCCL is resolved at run time from the libnccl.so.2 the process
 * has loaded (PyTorch's); rank 0 creates n_comms (1 or 2) ids (dm_nccl_unique_id), the caller
 * distributes the n_comms x 128 bytes (e.g. torch.distributed.broadcast) and every rank calls
 * dm_nccl_init.  With two communicators consecutive windows alternate between them, so that --
 * called on alternating streams -- two all-reduces are in flight.  This is the "one all-reduce
 * per window" of the multi-GPU configuration (BASELINE config 4). */
int dm_nccl_unique_id(uint8_t* out128);
int dm_nccl_init(dm_handle* h, const uint8_t* ids, uint32_t n_comms, uint32_t rank, uint32_t world);
int dm_window_allreduce(dm_handle* h, int with_keys, void* stream);
/* Statistics summed over all ranks as of the last dm_window_import, whatever stream it was enqueued on (this call and
 * dm_sync wait for it). */
int dm_get_global_stats(dm_handle* h, dm_stats_t* out);

/* Measurement support (bench.py): when enabled, every dm_process_lines records a CUDA
 * event pair on the launching stream around its dominant kernel (the tokenizer+detector
 * kernel).  dm_profile_read synchronises and returns the summed kernel time of the
 * launches timed since the last read, their count, and the total number of kernels this
 * handle has launched since dm_create. */
int dm_profile_enable(dm_handle* h, int on);
int dm_profile_read(dm_handle* h, double* kernel_ms_sum, uint64_t* n_timed, uint64_t* kernels_launched_total);

#ifdef __cplusplus
}
#endif
#endif /* DMDETECT_H */
