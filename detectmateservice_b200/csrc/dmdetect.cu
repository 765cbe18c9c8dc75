// dmdetect.cu -- host side of libdmdetect.so: the C ABI of include/dmdetect.h.
//
// Replaces, for one message of raw records, the Python call chain
//   Service.process -> CoreComponent.process -> NewValueDetector.train/detect
// (/root/reference/src/service/core.py:176-206; detector in the un-vendored
// detectmatelibrary).  No CPU path: every entry point that computes needs the device.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "dm_buf.h"
#include "dm_device.cuh"
#include "dm_kernels_index.cuh"
#include "dm_kernels_stream.cuh"
#include "dm_kernels_values.cuh"
#include "dm_kernels_records.cuh"
#include "dm_kernels_logs.cuh"
#include "dm_kernels_format.cuh"
#include "dm_kernels_lanes.cuh"
#include "dm_kernels_alerts.cuh"
#include "dm_kernels_parse.cuh"
#include "dm_kernels_window.cuh"
#include "dm_format_host.h"
#include "dm_host.h"

static void (*g_nccl_destroy_hook)(void*) = nullptr;   // set once NCCL is loaded (dm_nccl_load)

// ---------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int dm_fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define DM_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess)                                                               \
            return dm_fail(DM_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                           __FILE__, __LINE__);                                               \
    } while (0)

extern "C" const char* dm_last_error(void) { return g_err; }
extern "C" int dm_abi_version(void) { return DM_ABI_VERSION; }

extern "C" uint64_t dm_table_key(uint32_t field, const uint8_t* value, uint32_t len) {
    return dm_make_key(dm_fp64_bytes(value, len), dm_field_salt(field));
}

// ---------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------
struct dm_handle {
    int device = 0;
    int sm_count = 0;
    DmStream stream;                     // the handle's own stream
    cudaStream_t last_stream = nullptr;  // stream of the most recent enqueue
    uint64_t max_batch_bytes = 0, max_lines = 0;
    uint32_t table_log2 = 0;
    uint32_t n_keys = 0;
    int kernel_variant = 6;              // 6 = stream (default), 5 = lanes (one thread per record; DM_KERNEL=lanes)

    DmKeys h_keys;
    DmDev<DmKeys> d_keys;
    DmDev<uint8_t> d_in;                 // staging for host input
    DmDev<uint32_t> d_line_start;
    DmDev<uint8_t> d_flags;
    DmDev<float> d_scores;
    DmDev<DmBatchHeader> d_hdr;
    DmPinned<DmBatchHeader> h_hdr;
    DmPinned<unsigned int> h_err;        // the stream kernel's error word (DmxShared::error) as dm_sync last read it
    DmDev<dm_anomaly_t> d_anoms;
    uint32_t anomaly_cap = 0;
    DmDev<unsigned long long> d_stats;   // 3 * DM_STATS_WORDS: own, exported, global
    unsigned long long* d_stats_exported = nullptr;
    unsigned long long* d_stats_global = nullptr;
    DmPinned<unsigned long long> h_stats;
    DmDev<unsigned long long> table_slots, table_novel, table_count;
    DmTable table;                       // the kernels' view of the three
    uint64_t novel_exported = 0;         // novel keys already shipped in a window
    uint64_t novel_pending = 0;          // novel keys the last window could not carry (more than DM_WINDOW_KEYS learnt)
    DmRowsScratch rows;                  // row / record index scratch (K_A: lanes and log_format kernels)
    DmxScratch dmx;                      // stream-variant scratch (default kernel)
    uint64_t last_nbytes = 0;
    DmDev<uint32_t> d_vals;              // record mode: offsets / fields / record_of
    DmDev<uint32_t> d_masks;
    DmDev<DmMonitors> d_mons;            // record mode on the device
    bool mons_set = false;
    DmMonitors h_mons;             // host copy (dm_set_monitors + dm_set_combos)
    DmDev<DmFormat> d_fmt;         // log_format + templates (dm_set_format)
    DmDev<uint8_t> d_norm;         // R-norm: the message's normalised Content text (dm_set_format_ex with flags)
    bool fmt_norm = false;         // R-norm runs (dm_format_norm)
    void* nccl_comm[2] = {nullptr, nullptr};   // own NCCL communicators (dm_nccl_init): windows alternate between them
    uint32_t nccl_n = 0, nccl_rank = 0, nccl_world = 1;
    DmDev<unsigned long long> d_win[2];  // window exchange buffers of dm_window_allreduce
    DmEvent ev_win_done[2];
    uint64_t win_seq = 0;
    DmEvent ev_import;                   // recorded by every dm_window_import, on whichever stream it ran
    DmEvent ev_order;                    // dm_use_stream: the previous stream's work, waited for by the next stream
    bool fmt_set = false;
    uint32_t fmt_slots = 1;        // DmFormat.max_slots (dynamic shared memory of the thread-per-record kernel)
    // LogSchema input (dm_process_logs), allocated on first use
    DmDev<uint8_t> d_logs_text;          // the compacted texts + slack
    DmDev<uint8_t> d_logs;               // per-record / per-line / per-chunk arrays of DmLogsArgs
    uint64_t logs_cap = 0;               // records they hold
    uint32_t logs_chunks = 0;            // chunks they hold
    DmDev<DmLogsHeader> d_lhdr;
    DmPinned<DmLogsHeader> h_lhdr;
    // DetectorSchema alerts on the device (dm_set_alert_format / dm_encode_alerts), allocated by dm_set_alert_format
    const uint8_t* last_buf = nullptr;   // the last dm_process_lines batch as its kernels read it, and its scores
    const float* last_scores = nullptr;
    uint32_t last_src = DMA_SRC_NONE;    // where the last batch came from: what dm_encode_alerts can word
    uint32_t last_n_records = 0;         // its records (dm_process_records)
    DmDev<DmAlertFmt> d_afmt;
    DmDev<DmAlertHeader> d_ahdr;
    DmPinned<DmAlertHeader> h_ahdr;
    DmDev<uint8_t> d_alert;              // rank (max_lines + 1), per anomalous record line / mask / offset / size, tile sums
    DmDev<uint8_t> d_aout;               // the encoded alerts
    uint32_t alert_time_cap = DMA_NONE;  // log_format mode: the header capture named Time
    std::unique_ptr<DmFormat> h_fmt;     // host copy of the last dm_set_format[_ex] format (the encoder's is built from it)
    DmDev<DmFormat> d_efmt;              // the encoder's format: h_fmt keeping the Time capture too (dm_alert_efmt_build)
    uint32_t efmt_slots = 1;
    // the MatcherParser stage (dm_set_parser_format / dm_parse_logs)
    DmDev<DmParseFmt> d_pf;
    DmDev<DmFormat> d_pfmt;              // h_fmt keeping every capture (dm_parse_efmt_build)
    uint32_t pfmt_slots = 1;
    bool parse_set = false;              // cleared by dm_set_format[_ex]: the parser's format is built from h_fmt
    DmDev<unsigned long long> d_psize;   // per record its size, then the scan's tile sums and total
    DmDev<uint8_t> d_pout;               // the ParserSchemas, and their host copy
    DmPinned<uint8_t> h_pout;
    DmPinned<unsigned long long> h_ptotal;
    // pipelined host path: two slots
    struct Slot {
        DmDev<uint8_t> d_in; DmDev<uint8_t> d_flags; DmDev<float> d_scores;
        DmDev<DmBatchHeader> d_hdr; DmPinned<DmBatchHeader> h_hdr; DmDev<dm_anomaly_t> d_anoms;
        DmPinned<uint8_t> h_flags; DmPinned<float> h_scores;
        DmEvent ev_in, ev_comp, ev_hdr;
        DmStream st_out;
        bool busy = false;
    } slots[2];
    DmStream st_in;
    bool slots_ready = false;
    // measurement support
    bool profile = false;
    std::vector<DmEvent> ev;             // pairs: ev[2i] start, ev[2i+1] stop
    size_t ev_used = 0;
    uint64_t launches = 0;               // kernels launched since dm_create
    // A last batch that dm_collect made (dm_encode_alerts): the slot's, for as long as last_src is DMA_LINES and
    // last_buf is that slot's input; every other call that makes or clears a last batch changes one of the two.
    int last_slot = -1;
    uint64_t slot_nbytes[2] = {0, 0};    // the message each slot was submitted last
    // dm_export_known's scratch (dm_known_scratch), allocated by the first export that finds a key
    DmDev<uint8_t> known_buf;
    DmKnownScratch known{};
    DmPinned<unsigned int> h_known_hist;    // the digit histograms and the compacted count
};

static const size_t DM_PROFILE_PAIRS = 4096;

static void dm_prof_mark(dm_handle* h, cudaStream_t st, int which) {
    if (!h->profile || h->ev_used / 2 >= DM_PROFILE_PAIRS) return;
    if (which == 0 && (h->ev_used & 1)) return;
    if (which == 1 && !(h->ev_used & 1)) return;
    cudaEventRecord(h->ev[h->ev_used].get(), st);
    h->ev_used++;
}

static void dm_prof_mark_cb(void* ctx, cudaStream_t st, int which) { dm_prof_mark((dm_handle*)ctx, st, which); }

static const uint32_t DM_WINDOW_KEYS = 1u << 16;    // keys one rank can ship per window

// Anything this library enqueues that is not a stream-variant detect launch ends the chain of
// overlapping launches on that stream: the next detect launch is then ordered behind it in full.
static void dm_break_chain(dm_handle* h, cudaStream_t st) {
    if (h->dmx.chain_stream == st) h->dmx.chain_stream = nullptr;
}

// Makes st the stream of the handle's next enqueue.  A call on another stream than the previous one first waits for
// the previous stream, and so for every earlier call: the handle's calls take effect in call order whatever streams
// they use, and waiting for last_stream waits for everything the handle enqueued.  A switch also ends the overlap
// chain.  Calls on one stream record and wait on nothing.
static int dm_use_stream(dm_handle* h, cudaStream_t st) {
    if (st == h->last_stream) return DM_OK;
    DM_CUDA(cudaEventRecord(h->ev_order.get(), h->last_stream));
    DM_CUDA(cudaStreamWaitEvent(st, h->ev_order.get(), 0));
    h->last_stream = st;
    h->dmx.chain_stream = nullptr;
    return DM_OK;
}

static int dm_pick_stream(dm_handle* h, void* stream, cudaStream_t* out) {
    *out = stream ? (cudaStream_t)stream : h->stream.get();
    return dm_use_stream(h, *out);
}

extern "C" int dm_destroy(dm_handle* h);
// Everything dm_create allocates; on failure dm_create frees whatever was allocated so far (dm_destroy).
static int dm_create_fill(dm_handle* h, int device, const cudaDeviceProp& prop, uint32_t n_keys, const uint8_t* keys_blob,
                          const uint32_t* key_lens, uint64_t max_batch_bytes, uint64_t max_lines, uint32_t table_log2_slots) {
    h->device = device;
    h->sm_count = prop.multiProcessorCount;
    h->max_batch_bytes = max_batch_bytes;
    h->max_lines = max_lines ? max_lines : std::max<uint64_t>(max_batch_bytes / 8, 1024);
    h->table_log2 = table_log2_slots;
    h->n_keys = n_keys;
    memset(&h->h_keys, 0, sizeof(DmKeys));
    h->h_keys.n = n_keys;
    uint64_t off = 0;
    for (uint32_t k = 0; k < n_keys; ++k) {
        uint32_t len = key_lens[k];
        if (len == 0 || len > DM_MAX_KEYLEN) { return dm_fail(DM_ERR_ARG, "key %u: length %u not in 1..%d", k, len, DM_MAX_KEYLEN); }
        for (uint32_t i = 0; i < len; ++i) {
            uint8_t c = keys_blob[off + i];
            if (c == 0x20 || c == 0x22 || c == 0x27 || c == 0x3D || c == 0x0A) { return dm_fail(DM_ERR_ARG, "key %u holds a separator byte 0x%02x", k, c); }
            h->h_keys.bytes[k][i] = c;
        }
        for (uint32_t j = 0; j < k; ++j)
            if (h->h_keys.len[j] == len && memcmp(h->h_keys.bytes[j], h->h_keys.bytes[k], len) == 0) { return dm_fail(DM_ERR_ARG, "key %u duplicates key %u", k, j); }
        h->h_keys.len[k] = len;
        h->h_keys.salt[k] = dm_field_salt(k);
        off += len;
    }
    dm_keys_finalize_host(&h->h_keys);

    DM_CUDA(h->stream.create());
    h->last_stream = h->stream.get();
    DM_CUDA(dm_upload(h->d_keys, h->h_keys, h->last_stream));
    DM_CUDA(h->d_in.alloc(max_batch_bytes + 256, true));
    DM_CUDA(h->d_line_start.alloc(h->max_lines + 2));
    DM_CUDA(h->d_flags.alloc(h->max_lines + 16));
    DM_CUDA(h->d_scores.alloc(h->max_lines + 4));
    DM_CUDA(h->d_hdr.alloc(1, true));
    DM_CUDA(h->h_hdr.alloc(1, true));
    DM_CUDA(h->h_err.alloc(1, true));
    h->anomaly_cap = (uint32_t)std::min<uint64_t>(h->max_lines, 1u << 20);
    DM_CUDA(h->d_anoms.alloc(h->anomaly_cap));
    DM_CUDA(h->d_stats.alloc(3 * DM_STATS_WORDS, true));
    h->d_stats_exported = h->d_stats.get() + DM_STATS_WORDS;
    h->d_stats_global = h->d_stats.get() + 2 * DM_STATS_WORDS;
    DM_CUDA(h->h_stats.alloc(DM_STATS_WORDS));
    DM_CUDA(h->ev_import.create());
    DM_CUDA(h->ev_order.create());

    const uint64_t cap = 1ull << table_log2_slots;
    h->table.mask = (uint32_t)(cap - 1);
    h->table.limit = (uint32_t)(cap / 2);
    h->table.novel_cap = (uint32_t)(cap / 2);
    DM_CUDA(h->table_slots.alloc(cap, true));
    DM_CUDA(h->table_novel.alloc(cap / 2));
    DM_CUDA(h->table_count.alloc(2, true));
    h->table.slots = h->table_slots.get();
    h->table.novel = h->table_novel.get();
    h->table.count = h->table_count.get();
    h->table.novel_count = h->table.count + 1;

    int rc = dm_rows_scratch_create(&h->rows, max_batch_bytes, h->sm_count);
    if (rc != DM_OK) { return dm_fail(DM_ERR_CUDA, "row index scratch allocation failed: %s", cudaGetErrorString(cudaGetLastError())); }
    rc = dmx_scratch_create(&h->dmx, h->h_keys, max_batch_bytes, h->anomaly_cap, h->sm_count, h->last_stream);
    if (rc == DM_ERR_ARG) return dm_fail(DM_ERR_ARG, "DM_STREAM_RECHECK=%s: thread, chain or auto", getenv("DM_STREAM_RECHECK"));
    if (rc != DM_OK) { return dm_fail(DM_ERR_CUDA, "stream scratch allocation failed: %s", cudaGetErrorString(cudaGetLastError())); }
    { const char* ov = getenv("DM_OVERLAP"); if (ov) h->dmx.overlap = atoi(ov) != 0; }
    const char* env = getenv("DM_KERNEL");
    if (env && env[0]) {
        if (strcmp(env, "lanes") == 0) h->kernel_variant = 5;
        else if (strcmp(env, "stream") == 0) h->kernel_variant = 6;
        else return dm_fail(DM_ERR_ARG, "DM_KERNEL=%s: the key=value kernels are 'stream' (default) and 'lanes'", env);
    }
    DM_CUDA(cudaDeviceSynchronize());
    return DM_OK;
}


extern "C" int dm_create(int device, uint32_t n_keys, const uint8_t* keys_blob, const uint32_t* key_lens,
                         uint64_t max_batch_bytes, uint64_t max_lines, uint32_t table_log2_slots,
                         dm_handle** out) {
    if (!out) return dm_fail(DM_ERR_ARG, "out is NULL");
    *out = nullptr;
    if (n_keys > DM_MAX_KEYS) return dm_fail(DM_ERR_ARG, "n_keys %u > %d", n_keys, DM_MAX_KEYS);
    if (n_keys && (!keys_blob || !key_lens)) return dm_fail(DM_ERR_ARG, "keys missing");
    if (max_batch_bytes == 0 || max_batch_bytes > 0xFFFFFF00ull)
        return dm_fail(DM_ERR_ARG, "max_batch_bytes must be in 1..2^32-256");
    if (table_log2_slots < 10 || table_log2_slots > 28)
        return dm_fail(DM_ERR_ARG, "table_log2_slots must be in 10..28");
    int n_dev = 0;
    cudaError_t ce = cudaGetDeviceCount(&n_dev);
    if (ce != cudaSuccess || n_dev <= 0)
        return dm_fail(DM_ERR_NO_DEVICE, "no CUDA device (%s); this library has no CPU path",
                       ce == cudaSuccess ? "device count 0" : cudaGetErrorString(ce));
    if (device < 0 || device >= n_dev) return dm_fail(DM_ERR_ARG, "device %d out of range (0..%d)", device, n_dev - 1);
    cudaDeviceProp prop;
    DM_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)          // sm_90a code loads on compute capability 9.0 only
        return dm_fail(DM_ERR_NO_DEVICE, "device %d is sm_%d%d; libdmdetect is built for sm_90a (H100) only", device,
                       prop.major, prop.minor);
    DM_CUDA(cudaSetDevice(device));

    dm_handle* h = new (std::nothrow) dm_handle();
    if (!h) return dm_fail(DM_ERR_ARG, "out of host memory");
    const int rc = dm_create_fill(h, device, prop, n_keys, keys_blob, key_lens, max_batch_bytes, max_lines, table_log2_slots);
    if (rc != DM_OK) {
        dm_destroy(h);                                       // (sets no error message)
        return rc;
    }
    *out = h;
    return DM_OK;
}

extern "C" int dm_set_overlap(dm_handle* h, int on) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    h->dmx.overlap = on != 0;
    h->dmx.chain_stream = nullptr;
    return DM_OK;
}

extern "C" int dm_profile_enable(dm_handle* h, int on) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    DM_CUDA(cudaSetDevice(h->device));
    if (on && h->ev.empty()) {
        h->ev.resize(2 * DM_PROFILE_PAIRS);
        for (auto& e : h->ev) DM_CUDA(e.create(cudaEventDefault));
    }
    h->profile = on != 0;
    h->ev_used = 0;
    return DM_OK;
}

extern "C" int dm_profile_read(dm_handle* h, double* kernel_ms_sum, uint64_t* n_timed, uint64_t* kernels_launched_total) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(cudaStreamSynchronize(h->last_stream));
    double sum = 0.0;
    const size_t pairs = h->ev_used / 2;
    for (size_t i = 0; i < pairs; ++i) {
        float ms = 0.f;
        DM_CUDA(cudaEventElapsedTime(&ms, h->ev[2 * i].get(), h->ev[2 * i + 1].get()));
        sum += ms;
    }
    h->ev_used = 0;
    if (kernel_ms_sum) *kernel_ms_sum = sum;
    if (n_timed) *n_timed = pairs;
    if (kernels_launched_total) *kernels_launched_total = h->launches;
    return DM_OK;
}

// The handle's members free what they own when it is deleted: on its device, after everything it enqueued.
extern "C" int dm_destroy(dm_handle* h) {
    if (!h) return DM_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (void* comm : h->nccl_comm)
        if (comm && g_nccl_destroy_hook) g_nccl_destroy_hook(comm);
    delete h;
    return DM_OK;
}

static int dm_check_device_errors(dm_handle* h) {
    unsigned int err = h->h_hdr.get()->error;
    if (h->h_hdr.get()->anomaly_list_count > h->anomaly_cap) err |= DM_DEVERR_ANOMALY_OVERFLOW;
    if (err & DM_DEVERR_TABLE_FULL)
        return dm_fail(DM_ERR_TABLE_FULL, "known-set table over its load limit (2^%u slots); recreate with a larger table_log2_slots", h->table_log2);
    if (err & DM_DEVERR_NOVEL_OVERFLOW)
        return dm_fail(DM_ERR_TABLE_FULL, "more than %u distinct values learnt; novel-key list full", h->table.novel_cap);
    if (err & DM_DEVERR_ANOMALY_OVERFLOW)
        return dm_fail(DM_ERR_CAPACITY, "more than %u unknown values in one batch; the anomaly list is full", h->anomaly_cap);
    if (err & DM_DEVERR_TOO_MANY_LINES)
        return dm_fail(DM_ERR_CAPACITY, "batch holds more than max_lines=%llu records", (unsigned long long)h->max_lines);
    return DM_OK;
}

// The header only holds the last message's errors; the stream kernel ORs those of every message enqueued by
// dm_process_lines into the handle's error word as well.  Enqueues on st the copy of that word to h_err and its
// clearing: after st is synchronised, dm_header_with_errors folds it into h_hdr.
static int dm_fetch_errors(dm_handle* h, cudaStream_t st) {
    DM_CUDA(cudaMemcpyAsync(h->h_err.get(), &h->dmx.d_shared.get()->error, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaMemsetAsync(&h->dmx.d_shared.get()->error, 0, sizeof(unsigned int), st));
    return DM_OK;
}

static int dm_header_with_errors(dm_handle* h) {
    h->h_hdr.get()->error |= *h->h_err.get();
    *h->h_err.get() = 0;
    return dm_check_device_errors(h);
}

// ---------------------------------------------------------------------------------------
// the hot path
// ---------------------------------------------------------------------------------------
extern "C" int dm_process_lines(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int buf_on_device,
                                uint64_t n_train_lines, uint8_t* flags_out, float* scores_out,
                                uint64_t out_cap_lines, int out_on_device, uint64_t* n_lines_out,
                                uint64_t* n_anomalies_out, void* stream_) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (nbytes > h->max_batch_bytes)
        return dm_fail(DM_ERR_CAPACITY, "message of %llu bytes exceeds max_batch_bytes=%llu", (unsigned long long)nbytes, (unsigned long long)h->max_batch_bytes);
    if (nbytes && !buf) return dm_fail(DM_ERR_ARG, "buf is NULL");
    if (buf_on_device && (((uintptr_t)buf) & 15)) return dm_fail(DM_ERR_ARG, "device buf must be 16-byte aligned");
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st;
    const int rc_st = dm_pick_stream(h, stream_, &st);
    if (rc_st != DM_OK) return rc_st;

    const uint8_t* d_buf = buf;
    if (!buf_on_device) {
        if (nbytes) DM_CUDA(cudaMemcpyAsync(h->d_in.get(), buf, nbytes, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemsetAsync(h->d_in.get() + nbytes, 0, 64, st));
        d_buf = h->d_in.get();
    }
    const bool host_out = !out_on_device && (flags_out || scores_out);
    uint8_t* d_flags = (out_on_device && flags_out) ? flags_out : h->d_flags.get();
    float* d_scores = (out_on_device && scores_out) ? scores_out : h->d_scores.get();
    // when only one of the two outputs is a caller device buffer the other stays internal
    const uint64_t cap_flags = (out_on_device && flags_out) ? out_cap_lines : h->max_lines;
    const uint64_t cap_scores = (out_on_device && scores_out) ? out_cap_lines : h->max_lines;
    const uint64_t out_cap = std::min(cap_flags, cap_scores);

    bool stream_kernel = false;
    // (the stream kernel and K_A write the per-batch header themselves)
    if (nbytes == 0) DM_CUDA(cudaMemsetAsync(h->d_hdr.get(), 0, sizeof(DmBatchHeader), st));
    h->last_nbytes = nbytes;

    if (h->fmt_set) {
        // log_format / template mode: K_A writes the record index, then one THREAD per record
        if ((nbytes + DMR_ROW - 1) / DMR_ROW > h->rows.max_rows) return dm_fail(DM_ERR_CAPACITY, "message too large for the row index");
        const DmRowsArgs ra = dm_rows_args(d_buf, nbytes, h->rows.d_row_prefix.get(), h->rows.d_tile_state.get(), &h->rows.epoch, h->d_line_start.get(),
                                           d_flags, d_scores, out_cap, h->d_hdr.get(), h->d_stats.get(), n_train_lines, h->max_lines);
        if (ra.n_rows > 0) {
            dm_launch_pdl(dm_k_rowindex, ra.n_tiles, DMR_A_THREADS, st, h->rows.pdl, ra);
            // combination monitors: the COMBO instantiations re-hash their members from the captures the lanes keep
            const bool combos = h->mons_set && h->h_mons.n_combos > 0;
            DmDetectArgs a = dm_detect_args(d_buf, nbytes, h->d_line_start.get(), h->d_hdr.get(), h->d_keys.get(), h->table, d_flags, d_scores, out_cap,
                                            h->d_anoms.get(), h->anomaly_cap, h->d_stats.get(), combos ? (const void*)h->d_mons.get() : nullptr);
            const unsigned grid = dm_detect_grid(nbytes, h->max_lines, DM_FMTL_THREADS, (uint64_t)h->sm_count * 32);
            const size_t smem = (size_t)2 * h->fmt_slots * DM_FMTL_THREADS * sizeof(uint2);
            const bool norm = h->fmt_norm;
            if (n_train_lines > 0) {
                a.line_lo = 0; a.line_hi = n_train_lines;
                dm_launch_pdl_smem(dm_format_lanes_kernel(true, norm, combos), grid, DM_FMTL_THREADS, smem, st, false, a,
                                   (const DmFormat*)h->d_fmt.get(), h->d_norm.get());
            }
            a.line_lo = n_train_lines; a.line_hi = ~0ull;
            dm_prof_mark(h, st, 0);
            dm_launch_pdl_smem(dm_format_lanes_kernel(false, norm, combos), grid, DM_FMTL_THREADS, smem, st, false, a,
                               (const DmFormat*)h->d_fmt.get(), h->d_norm.get());
            dm_prof_mark(h, st, 1);
            h->launches += 2 + (n_train_lines > 0 ? 1 : 0);
        }
    } else if (h->kernel_variant == 5 || (h->mons_set && h->h_mons.n_combos > 0)) {
        // one thread per record; the only raw-line kernel that evaluates combination monitors
        const bool combos = h->mons_set && h->h_mons.n_combos > 0;
        const int rc = dm_lanes_launch(&h->rows, h->d_line_start.get(), d_buf, nbytes, n_train_lines, h->d_keys.get(), h->table, d_flags,
                                       d_scores, out_cap, h->d_anoms.get(), h->anomaly_cap, h->d_hdr.get(), h->d_stats.get(), h->max_lines,
                                       h->sm_count, combos ? (const void*)h->d_mons.get() : nullptr, h->n_keys, st, dm_prof_mark_cb, h);
        if (rc < 0) return dm_fail(DM_ERR_CUDA, "lanes kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        h->launches += (uint64_t)rc;
    } else {
        stream_kernel = true;
        const int rc = dmx_launch(&h->dmx, d_buf, nbytes, n_train_lines, h->table, d_flags, d_scores, out_cap, h->d_anoms.get(),
                                  h->anomaly_cap, h->d_hdr.get(), h->d_stats.get(), h->max_lines, st, h->dmx.overlap, true, dm_prof_mark_cb, h);
        if (rc < 0) return dm_fail(DM_ERR_CUDA, "stream kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        h->launches += (uint64_t)rc;
    }
    DM_CUDA(cudaGetLastError());
    if (!stream_kernel) h->dmx.chain_stream = nullptr;     // (a launch that is not the stream kernel's ends the overlap chain)
    h->last_buf = d_buf;
    h->last_scores = d_scores;
    h->last_src = DMA_LINES;

    const bool want_sync = host_out || n_lines_out || n_anomalies_out;
    if (!want_sync) return DM_OK;

    DM_CUDA(cudaMemcpyAsync(h->h_hdr.get(), h->d_hdr.get(), sizeof(DmBatchHeader), cudaMemcpyDeviceToHost, st));
    int rc = dm_fetch_errors(h, st);
    if (rc != DM_OK) return rc;
    DM_CUDA(cudaStreamSynchronize(st));
    rc = dm_header_with_errors(h);
    if (rc != DM_OK) return rc;
    const uint64_t n_lines = h->h_hdr.get()->n_lines;
    if (n_lines_out) *n_lines_out = n_lines;
    if (n_anomalies_out) *n_anomalies_out = h->h_hdr.get()->n_anomalies;
    if (host_out) {
        if (n_lines > out_cap_lines)
            return dm_fail(DM_ERR_CAPACITY, "batch holds %llu records, output capacity is %llu", (unsigned long long)n_lines, (unsigned long long)out_cap_lines);
        if (flags_out && n_lines) DM_CUDA(cudaMemcpyAsync(flags_out, h->d_flags.get(), n_lines, cudaMemcpyDeviceToHost, st));
        if (scores_out && n_lines) DM_CUDA(cudaMemcpyAsync(scores_out, h->d_scores.get(), n_lines * sizeof(float), cudaMemcpyDeviceToHost, st));
        DM_CUDA(cudaStreamSynchronize(st));
    }
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// record mode
// ---------------------------------------------------------------------------------------
// Adds what a synchronous record call counts on the host (dm_stats_add_records) to the handle's statistics.  The
// read-modify-write runs on the call's stream st: a copy on the legacy stream is not ordered against the handle's
// non-blocking streams, so a later kernel could add to d_stats before the write-back lands.
static int dm_records_stats(dm_handle* h, cudaStream_t st, uint64_t n_records, uint64_t trained, uint64_t scored, uint64_t nbytes) {
    unsigned long long cur[6];
    DM_CUDA(cudaMemcpyAsync(cur, h->d_stats.get(), sizeof(cur), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    dm_stats_add_records(cur, n_records, trained, scored, nbytes);
    DM_CUDA(cudaMemcpyAsync(h->d_stats.get(), cur, 3 * sizeof(cur[0]), cudaMemcpyHostToDevice, st));
    DM_CUDA(cudaMemcpyAsync(h->d_stats.get() + 5, &cur[5], sizeof(cur[5]), cudaMemcpyHostToDevice, st));
    DM_CUDA(cudaStreamSynchronize(st));
    return DM_OK;
}

extern "C" int dm_process_values(dm_handle* h, const uint8_t* blob, uint64_t blob_bytes, const uint32_t* offsets,
                                 const uint32_t* fields, const uint32_t* record_of, uint32_t n_values,
                                 uint32_t n_records, uint32_t n_train_records, uint64_t record_bytes,
                                 uint8_t* flags_out, float* scores_out, uint32_t* masks_out,
                                 uint64_t* n_anomalies_out) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (n_values && (!blob && blob_bytes)) return dm_fail(DM_ERR_ARG, "blob is NULL");
    if (n_values && (!offsets || !fields || !record_of)) return dm_fail(DM_ERR_ARG, "value arrays missing");
    if (blob_bytes > h->max_batch_bytes) return dm_fail(DM_ERR_CAPACITY, "value blob of %llu bytes exceeds max_batch_bytes", (unsigned long long)blob_bytes);
    if (n_records > h->max_lines) return dm_fail(DM_ERR_CAPACITY, "%u records exceed max_lines=%llu", n_records, (unsigned long long)h->max_lines);
    for (uint32_t i = 0; i < n_values; ++i) {
        if (fields[i] >= h->n_keys || record_of[i] >= n_records || offsets[i] > offsets[i + 1] || offsets[i + 1] > blob_bytes)
            return dm_fail(DM_ERR_ARG, "value %u: field/record/offset out of range", i);
    }
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream.get();
    int rc = dm_use_stream(h, st);
    if (rc != DM_OK) return rc;
    dm_break_chain(h, st);
    h->last_src = DMA_SRC_NONE;
    // d_vals holds 3 * vals_cap + 1 words: vals_cap + 1 offsets, vals_cap fields, vals_cap records
    if (n_values > h->d_vals.cap() / 3) DM_CUDA(h->d_vals.grow(3ull * n_values + 1, 3 * std::max<uint64_t>(2ull * n_values, 4096) + 1));
    DM_CUDA(h->d_masks.alloc(h->max_lines + 4));
    const uint64_t vals_cap = h->d_vals.cap() / 3;
    uint32_t* d_off = h->d_vals.get();
    uint32_t* d_fld = d_off + vals_cap + 1;
    uint32_t* d_rec = d_fld + vals_cap;
    DM_CUDA(cudaMemsetAsync(h->d_hdr.get(), 0, sizeof(DmBatchHeader), st));
    if (n_values) {
        if (blob_bytes) DM_CUDA(cudaMemcpyAsync(h->d_in.get(), blob, blob_bytes, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemcpyAsync(d_off, offsets, (uint64_t)(n_values + 1) * 4, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemcpyAsync(d_fld, fields, (uint64_t)n_values * 4, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemcpyAsync(d_rec, record_of, (uint64_t)n_values * 4, cudaMemcpyHostToDevice, st));
    }
    if (n_records) {
        DM_CUDA(cudaMemsetAsync(h->d_flags.get(), 0, n_records, st));
        DM_CUDA(cudaMemsetAsync(h->d_scores.get(), 0, (uint64_t)n_records * 4, st));
        DM_CUDA(cudaMemsetAsync(h->d_masks.get(), 0, (uint64_t)n_records * 4, st));
    }
    if (n_values) {
        DmValuesArgs a;
        a.blob = h->d_in.get(); a.offsets = d_off; a.fields = d_fld; a.record_of = d_rec; a.n_values = n_values;
        a.n_records = n_records; a.n_train_records = n_train_records; a.keys = h->d_keys.get(); a.table = h->table;
        a.flags = h->d_flags.get(); a.scores = h->d_scores.get(); a.masks = h->d_masks.get(); a.hdr = h->d_hdr.get(); a.stats = h->d_stats.get();
        const int grid = (int)std::min<uint32_t>((n_values + 255) / 256, (uint32_t)h->sm_count * 8);
        if (n_train_records > 0) { dm_k_values<<<grid, 256, 0, st>>>(a, 0); h->launches++; }
        dm_k_values<<<grid, 256, 0, st>>>(a, 1);
        h->launches++;
        DM_CUDA(cudaGetLastError());
    }
    DM_CUDA(cudaMemcpyAsync(h->h_hdr.get(), h->d_hdr.get(), sizeof(DmBatchHeader), cudaMemcpyDeviceToHost, st));
    if (flags_out && n_records) DM_CUDA(cudaMemcpyAsync(flags_out, h->d_flags.get(), n_records, cudaMemcpyDeviceToHost, st));
    if (scores_out && n_records) DM_CUDA(cudaMemcpyAsync(scores_out, h->d_scores.get(), (uint64_t)n_records * 4, cudaMemcpyDeviceToHost, st));
    if (masks_out && n_records) DM_CUDA(cudaMemcpyAsync(masks_out, h->d_masks.get(), (uint64_t)n_records * 4, cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    // statistics that do not need the device: record and byte counts
    const uint32_t tr = std::min<uint32_t>(n_train_records, n_records);
    rc = dm_records_stats(h, st, n_records, tr, n_records - tr, record_bytes);
    if (rc != DM_OK) return rc;
    h->h_hdr.get()->n_lines = n_records;
    rc = dm_check_device_errors(h);
    if (rc != DM_OK) return rc;
    if (n_anomalies_out) *n_anomalies_out = h->h_hdr.get()->n_anomalies;
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// record mode on the device (batches of length-delimited ParserSchema records)
// ---------------------------------------------------------------------------------------
static_assert(sizeof(dm_monitor_t) == sizeof(DmMonitor), "dm_monitor_t and DmMonitor must have the same layout");

extern "C" int dm_set_monitors(dm_handle* h, uint32_t n_monitors, const dm_monitor_t* monitors) {
    if (!h || (n_monitors && !monitors)) return dm_fail(DM_ERR_ARG, "NULL argument");
    if (n_monitors != h->n_keys) return dm_fail(DM_ERR_ARG, "%u monitors given, the handle was created with %u fields", n_monitors, h->n_keys);
    DmMonitors& hm = h->h_mons;
    memset(&hm, 0, sizeof(hm));
    hm.n = n_monitors;
    for (uint32_t i = 0; i < n_monitors; ++i) {
        if (monitors[i].source > 1) return dm_fail(DM_ERR_ARG, "monitor %u: source must be 0 (header) or 1 (variable)", i);
        if (monitors[i].source == 0 && (monitors[i].key_len == 0 || monitors[i].key_len > 64))
            return dm_fail(DM_ERR_ARG, "monitor %u: header key length %u not in 1..64", i, monitors[i].key_len);
        memcpy(&hm.m[i], &monitors[i], sizeof(DmMonitor));
    }
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(dm_upload(h->d_mons, hm, h->last_stream));
    h->mons_set = true;
    return DM_OK;
}

extern "C" int dm_set_combos(dm_handle* h, uint32_t n_combos, const uint32_t* member_off, const uint32_t* members,
                             uint32_t member_only_mask) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (!h->mons_set) return dm_fail(DM_ERR_STATE, "dm_set_monitors has not been called");
    if (n_combos && (!member_off || !members)) return dm_fail(DM_ERR_ARG, "NULL argument");
    DmMonitors& hm = h->h_mons;
    if (hm.n + n_combos > DM_MAX_KEYS)
        return dm_fail(DM_ERR_ARG, "%u monitors + %u combinations exceed the %d output-mask bits", hm.n, n_combos, DM_MAX_KEYS);
    if (n_combos && member_off[0] != 0) return dm_fail(DM_ERR_ARG, "member_off[0] must be 0");
    if (n_combos && member_off[n_combos] > DM_MAX_COMBO_MEMBERS)
        return dm_fail(DM_ERR_ARG, "%u combination members in total, at most %d", member_off[n_combos], DM_MAX_COMBO_MEMBERS);
    for (uint32_t c = 0; c < n_combos; ++c) {
        if (member_off[c + 1] <= member_off[c]) return dm_fail(DM_ERR_ARG, "combination %u is empty or member_off is not increasing", c);
        for (uint32_t j = member_off[c]; j < member_off[c + 1]; ++j)
            if (members[j] >= hm.n) return dm_fail(DM_ERR_ARG, "combination %u: member %u is not a monitor index (< %u)", c, members[j], hm.n);
    }
    if (hm.n < 32 && (member_only_mask >> hm.n)) return dm_fail(DM_ERR_ARG, "member_only_mask has bits beyond the %u monitors", hm.n);
    hm.n_combos = n_combos;
    hm.member_only = member_only_mask;
    memset(hm.combo_off, 0, sizeof(hm.combo_off));
    memset(hm.combo_members, 0, sizeof(hm.combo_members));
    for (uint32_t c = 0; c <= n_combos && n_combos; ++c) hm.combo_off[c] = member_off[c];
    for (uint32_t j = 0; n_combos && j < member_off[n_combos]; ++j) hm.combo_members[j] = (uint8_t)members[j];
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(dm_upload(h->d_mons, hm, h->last_stream));
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// log_format + templates (MatcherParser fused in front of the detector)
// ---------------------------------------------------------------------------------------

static int dm_alert_efmt_upload(dm_handle* h);

extern "C" int dm_set_format(dm_handle* h, const char* log_format, const char* content_name, uint32_t n_templates,
                             const char* const* templates) {
    return dm_set_format_ex(h, log_format, content_name, n_templates, templates, 0);
}

extern "C" int dm_set_format_ex(dm_handle* h, const char* log_format, const char* content_name, uint32_t n_templates,
                                const char* const* templates, uint32_t norm_flags) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (!log_format) {                                             // back to key=value tokenisation
        h->fmt_set = false;
        return DM_OK;
    }
    if (!h->mons_set) return dm_fail(DM_ERR_STATE, "dm_set_monitors has not been called");
    if (n_templates && !templates) return dm_fail(DM_ERR_ARG, "templates is NULL");
    std::unique_ptr<DmFormat> f(new (std::nothrow) DmFormat);
    if (!f) return dm_fail(DM_ERR_CUDA, "out of host memory");
    std::string err;
    if (!dm_format_build(log_format, content_name, n_templates, templates, norm_flags, h->h_mons, f.get(), &err))
        return dm_fail(DM_ERR_ARG, "%s", err.c_str());
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess && norm_flags && n_templates) e = h->d_norm.alloc(h->max_batch_bytes + 256);
    if (e == cudaSuccess) e = dm_upload(h->d_fmt, *f, h->last_stream);
    if (e != cudaSuccess) return dm_fail(DM_ERR_CUDA, "dm_set_format: %s", cudaGetErrorString(e));
    h->fmt_set = true;
    h->fmt_slots = f->max_slots;
    h->h_fmt = std::move(f);                                     // (kept: the alert encoder's format is built from it)
    h->fmt_norm = dm_format_norm(*h->h_fmt);
    h->parse_set = false;
    return dm_alert_efmt_upload(h);
}

extern "C" int dm_stream_recheck_chained(dm_handle* h) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    return h->dmx.last_chained ? 1 : 0;
}

// diagnostics: per-CTA time stamps of the last stream-kernel launch (DM_STREAM_TIMELINE=1)
extern "C" int dm_debug_rows_timeline(dm_handle* h, unsigned long long* out, uint64_t cap_words, uint32_t* n_warps_out) {
    if (!h || !n_warps_out) return dm_fail(DM_ERR_ARG, "NULL argument");
    if (h->dmx.d_timeline.get()) {
        // stream variant: per CTA {smid, t_start, t_rows_done, t_exit}, then 8 epilogue stamps
        *n_warps_out = h->dmx.last_grid;
        if (!out) return DM_OK;
        DM_CUDA(cudaSetDevice(h->device));
        DM_CUDA(cudaStreamSynchronize(h->last_stream));
        const uint64_t words = std::min<uint64_t>(cap_words, 4ull * h->dmx.last_grid + 8);
        DM_CUDA(cudaMemcpy(out, h->dmx.d_timeline.get(), words * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        return DM_OK;
    }
    return dm_fail(DM_ERR_STATE, "create the handle with DM_STREAM_TIMELINE=1");
}

// The error of a framing split (dm_frame_split).
static int dm_frame_fail(const DmFrames& f) {
    if (f.error == DM_FRAME_TRUNCATED) return dm_fail(DM_ERR_ARG, "truncated length prefix at byte %llu", (unsigned long long)f.at);
    return dm_fail(DM_ERR_ARG, "record of %llu bytes at byte %llu runs past the end of the message", (unsigned long long)f.rec_len,
                   (unsigned long long)f.at);
}

extern "C" int dm_process_records(dm_handle* h, const uint8_t* buf, uint64_t nbytes, uint32_t n_train_records,
                                  uint8_t* flags_out, float* scores_out, uint32_t* masks_out, uint64_t out_cap,
                                  uint64_t* n_records_out, uint64_t* n_anomalies_out) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (!h->mons_set) return dm_fail(DM_ERR_STATE, "dm_set_monitors has not been called");
    if (nbytes && !buf) return dm_fail(DM_ERR_ARG, "buf is NULL");
    if (nbytes > h->max_batch_bytes) return dm_fail(DM_ERR_CAPACITY, "message of %llu bytes exceeds max_batch_bytes=%llu", (unsigned long long)nbytes, (unsigned long long)h->max_batch_bytes);
    const DmFrames fr = dm_frame_split(buf, nbytes);
    if (fr.error) return dm_frame_fail(fr);
    const std::vector<uint32_t>& off = fr.off;
    const std::vector<uint32_t>& len = fr.len;
    const uint32_t n_records = (uint32_t)off.size();
    if (n_records > h->max_lines) return dm_fail(DM_ERR_CAPACITY, "%u records exceed max_lines=%llu", n_records, (unsigned long long)h->max_lines);
    if ((flags_out || scores_out || masks_out) && n_records > out_cap)
        return dm_fail(DM_ERR_CAPACITY, "batch holds %u records, output capacity is %llu", n_records, (unsigned long long)out_cap);
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream.get();
    int rc = dm_use_stream(h, st);
    if (rc != DM_OK) return rc;
    dm_break_chain(h, st);
    h->last_src = DMA_SRC_NONE;
    DM_CUDA(h->d_vals.grow(2ull * n_records + 2, 3 * std::max<uint64_t>(2ull * n_records, 4096) + 1));
    DM_CUDA(h->d_masks.alloc(h->max_lines + 4));
    uint32_t* d_off = h->d_vals.get();
    uint32_t* d_len = d_off + n_records;
    uint32_t* d_bound = d_off + 2ull * n_records;             // {first scored record, records trained}
    uint32_t bound[2] = {0, 0};
    DM_CUDA(cudaMemsetAsync(h->d_hdr.get(), 0, sizeof(DmBatchHeader), st));
    if (n_records) {
        // (every record writes its flag, score and mask in the train or the detect launch, malformed ones included)
        DM_CUDA(cudaMemcpyAsync(h->d_in.get(), buf, nbytes, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemcpyAsync(d_off, off.data(), (uint64_t)n_records * 4, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemcpyAsync(d_len, len.data(), (uint64_t)n_records * 4, cudaMemcpyHostToDevice, st));
        DmRecordsArgs a;
        a.buf = h->d_in.get(); a.rec_off = d_off; a.rec_len = d_len; a.n_records = n_records; a.n_train_records = n_train_records;
        a.mons = h->d_mons.get(); a.table = h->table; a.flags = h->d_flags.get(); a.scores = h->d_scores.get(); a.masks = h->d_masks.get();
        a.hdr = h->d_hdr.get(); a.stats = h->d_stats.get();
        const int grid = (int)std::min<uint32_t>((n_records + 127) / 128, (uint32_t)h->sm_count * 16);
        if (n_train_records > 0) {
            // training takes the first n_train_records WELL-FORMED records: mark them (flags as scratch), find the
            // bound, then insert.  Batches after training skip both extra launches.
            dm_k_records<<<grid, 128, 0, st>>>(a, 2);
            dm_k_records_bound<<<1, 256, 0, st>>>(h->d_flags.get(), n_records, n_train_records, d_bound);
            dm_k_records<<<grid, 128, 0, st>>>(a, 0, d_bound);
            h->launches += 3;
        }
        if (n_train_records < n_records) {
            dm_prof_mark(h, st, 0);
            dm_k_records<<<grid, 128, 0, st>>>(a, 1, n_train_records > 0 ? d_bound : nullptr);
            dm_prof_mark(h, st, 1);
            h->launches++;
        }
        DM_CUDA(cudaGetLastError());
    }
    DM_CUDA(cudaMemcpyAsync(h->h_hdr.get(), h->d_hdr.get(), sizeof(DmBatchHeader), cudaMemcpyDeviceToHost, st));
    if (flags_out && n_records) DM_CUDA(cudaMemcpyAsync(flags_out, h->d_flags.get(), n_records, cudaMemcpyDeviceToHost, st));
    if (scores_out && n_records) DM_CUDA(cudaMemcpyAsync(scores_out, h->d_scores.get(), (uint64_t)n_records * 4, cudaMemcpyDeviceToHost, st));
    if (masks_out && n_records) DM_CUDA(cudaMemcpyAsync(masks_out, h->d_masks.get(), (uint64_t)n_records * 4, cudaMemcpyDeviceToHost, st));
    if (n_records && n_train_records > 0) DM_CUDA(cudaMemcpyAsync(bound, d_bound, sizeof(bound), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    // train_lines: the records trained; detect_lines: the records from the bound on (malformed ones included)
    const uint64_t first_scored = n_train_records > 0 ? bound[0] : 0;
    rc = dm_records_stats(h, st, n_records, bound[1], n_records - first_scored, nbytes);
    if (rc != DM_OK) return rc;
    h->h_hdr.get()->n_lines = n_records;
    rc = dm_check_device_errors(h);
    if (rc != DM_OK) return rc;
    if (n_records_out) *n_records_out = n_records;
    if (n_anomalies_out) *n_anomalies_out = h->h_hdr.get()->n_anomalies;
    h->last_src = DMA_RECORDS;
    h->last_n_records = n_records;
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// LogSchema input (the reader stage's records): unwrapped on the device, then the line path
// ---------------------------------------------------------------------------------------
// The compacted texts (dm_logs_text_bytes): one buffer, allocated on the first call, serves every call.  The
// per-record arrays (dm_logs_scratch_bytes) grow with the largest batch seen; they hold `chunks` walk chunks, the most
// any of the handle's walk plans makes.
static int dm_logs_reserve(dm_handle* h, uint64_t n_records, uint32_t chunks) {
    if (!h->d_lhdr.get()) {                                          // (kept only when all three were allocated)
        DmDev<DmLogsHeader> d_lhdr; DmPinned<DmLogsHeader> h_lhdr; DmDev<uint8_t> text;
        DM_CUDA(d_lhdr.alloc(1));
        DM_CUDA(h_lhdr.alloc(1));
        DM_CUDA(text.alloc(dm_logs_text_bytes(h->max_batch_bytes)));
        h->d_lhdr = std::move(d_lhdr);
        h->h_lhdr = std::move(h_lhdr);
        h->d_logs_text = std::move(text);
    }
    if (n_records <= h->logs_cap) return DM_OK;
    const uint64_t cap = std::min<uint64_t>(std::max<uint64_t>({n_records, 2 * h->logs_cap, 4096}), h->max_lines);
    const uint64_t bytes = dm_logs_scratch_bytes(cap, chunks);
    h->logs_cap = 0;
    DM_CUDA(h->d_logs.grow(bytes, bytes));
    h->logs_cap = cap;
    h->logs_chunks = chunks;
    return DM_OK;
}

// The records of a LogSchema message (one bare record, or varint length, payload, varint length, payload ...), refused
// where the framing is broken or they exceed max_lines.
static int dm_logs_frames(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int delimited, DmFrames* fr) {
    *fr = dm_frame_records(buf, nbytes, delimited != 0);
    if (fr->error) return dm_frame_fail(*fr);
    const uint32_t n_records = (uint32_t)fr->off.size();
    if (n_records > h->max_lines) return dm_fail(DM_ERR_CAPACITY, "%u records exceed max_lines=%llu", n_records, (unsigned long long)h->max_lines);
    return DM_OK;
}

// Enqueues the message's copy to the device and the unwrap kernels on the handle's stream, up to and including the copy
// of the header the host reads back (h_lhdr; not synchronised).  copy: also compact the texts into d_logs_text for the
// line path; without it the per-record text bounds and ranks are all that is computed.
static int dm_logs_unwrap(dm_handle* h, const uint8_t* buf, uint64_t nbytes, const DmFrames& fr, uint32_t n_train_records,
                          bool copy, DmLogsArgs* out, float** d_rscores, uint8_t** d_rflags) {
    const uint32_t n_records = (uint32_t)fr.off.size();
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream.get();
    int rc = dm_use_stream(h, st);
    if (rc != DM_OK) return rc;
    dm_break_chain(h, st);
    // walk grid: at most 4 CTAs per SM
    const uint32_t walk_ctas = (uint32_t)h->sm_count * 4;
    rc = dm_logs_reserve(h, n_records, walk_ctas);
    if (rc != DM_OK) return rc;
    DmLogsArgs a = dm_logs_carve(h->d_logs.get(), h->logs_cap, h->logs_chunks, h->d_lhdr.get(), d_rscores, d_rflags);
    dm_logs_call(&a, h->d_in.get(), n_records, n_train_records, walk_ctas, copy ? h->d_logs_text.get() : nullptr,
                 copy ? h->d_logs_text.cap() : 0);
    if (nbytes) DM_CUDA(cudaMemcpyAsync(h->d_in.get(), buf, nbytes, cudaMemcpyHostToDevice, st));
    if (n_records) {
        DM_CUDA(cudaMemcpyAsync((void*)a.rec_off, fr.off.data(), (uint64_t)n_records * 4, cudaMemcpyHostToDevice, st));
        DM_CUDA(cudaMemcpyAsync((void*)a.rec_len, fr.len.data(), (uint64_t)n_records * 4, cudaMemcpyHostToDevice, st));
        dm_k_logs_walk<<<a.n_chunks, DML_THREADS, 0, st>>>(a);
        dm_k_logs_scan<<<1, DML_THREADS, 0, st>>>(a);
        dm_k_logs_compact<<<dm_grid(n_records, DML_THREADS, (uint64_t)h->sm_count * 8), DML_THREADS, 0, st>>>(a);
        h->launches += 3;
        if (copy) {
            dm_k_logs_copy<<<dm_logs_copy_grid(nbytes, (uint64_t)h->sm_count * 16), DML_THREADS, 0, st>>>(a);
            h->launches++;
        }
        DM_CUDA(cudaGetLastError());
    } else {
        DM_CUDA(cudaMemsetAsync(h->d_lhdr.get(), 0, sizeof(DmLogsHeader), st));
    }
    DM_CUDA(cudaMemcpyAsync(h->h_lhdr.get(), h->d_lhdr.get(), sizeof(DmLogsHeader), cudaMemcpyDeviceToHost, st));
    *out = a;
    return DM_OK;
}

extern "C" int dm_process_logs(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int delimited, uint32_t n_train_records,
                               uint8_t* flags_out, float* scores_out, uint64_t out_cap,
                               uint64_t* n_records_out, uint64_t* n_malformed_out, uint64_t* n_anomalies_out) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (nbytes && !buf) return dm_fail(DM_ERR_ARG, "buf is NULL");
    if (nbytes > h->max_batch_bytes) return dm_fail(DM_ERR_CAPACITY, "message of %llu bytes exceeds max_batch_bytes=%llu", (unsigned long long)nbytes, (unsigned long long)h->max_batch_bytes);
    DmFrames fr;
    int rc = dm_logs_frames(h, buf, nbytes, delimited, &fr);
    if (rc != DM_OK) return rc;
    const uint32_t n_records = (uint32_t)fr.off.size();
    if ((flags_out || scores_out) && n_records > out_cap)
        return dm_fail(DM_ERR_CAPACITY, "batch holds %u records, output capacity is %llu", n_records, (unsigned long long)out_cap);
    DmLogsArgs a;
    float* d_rscores;
    uint8_t* d_rflags;
    rc = dm_logs_unwrap(h, buf, nbytes, fr, n_train_records, true, &a, &d_rscores, &d_rflags);
    if (rc != DM_OK) return rc;
    cudaStream_t st = h->stream.get();
    DM_CUDA(cudaStreamSynchronize(st));
    const DmLogsHeader lh = *h->h_lhdr.get();
    if (lh.n_lines) {
        uint64_t n_lines = 0, n_anoms = 0;
        rc = dm_process_lines(h, h->d_logs_text.get(), lh.total_bytes, 1, lh.n_train, nullptr, nullptr, 0, 0, &n_lines, &n_anoms, st);
        dm_break_chain(h, st);
        h->last_src = DMA_SRC_NONE;                           // (its anomaly list is rewritten to records below)
        if (rc != DM_OK) return rc;
        if (n_lines != lh.n_lines)
            return dm_fail(DM_ERR_STATE, "the line path found %llu records in %llu unwrapped texts", (unsigned long long)n_lines, (unsigned long long)lh.n_lines);
    } else {
        DM_CUDA(cudaMemsetAsync(h->d_hdr.get(), 0, sizeof(DmBatchHeader), st));
        h->last_src = DMA_SRC_NONE;
    }
    const unsigned grid_s = dm_logs_scatter_grid(n_records, h->anomaly_cap, (uint64_t)h->sm_count * 8);
    dm_k_logs_scatter<<<grid_s, DML_THREADS, 0, st>>>(a, h->d_flags.get(), h->d_scores.get(), d_rflags, d_rscores, h->d_anoms.get(), h->anomaly_cap,
                                                     h->d_hdr.get(), h->d_stats.get(), nbytes);
    h->launches++;
    DM_CUDA(cudaGetLastError());
    DM_CUDA(cudaMemcpyAsync(h->h_hdr.get(), h->d_hdr.get(), sizeof(DmBatchHeader), cudaMemcpyDeviceToHost, st));
    if (flags_out && n_records) DM_CUDA(cudaMemcpyAsync(flags_out, d_rflags, n_records, cudaMemcpyDeviceToHost, st));
    if (scores_out && n_records) DM_CUDA(cudaMemcpyAsync(scores_out, d_rscores, (uint64_t)n_records * 4, cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    if (n_records_out) *n_records_out = n_records;
    if (n_malformed_out) *n_malformed_out = n_records - lh.n_lines;
    if (n_anomalies_out) *n_anomalies_out = h->h_hdr.get()->n_anomalies;
    h->last_src = DMA_LOGS;                                   // (the line path left last_buf / last_nbytes: the texts)
    h->last_scores = d_rscores;
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// DetectorSchema alerts of raw-line batches, encoded on the device (dm_kernels_alerts.cuh)
// ---------------------------------------------------------------------------------------
// The encoder's copy of the log_format (when both the format and the alert format are set): the matcher's own, keeping
// the Time capture as well.
static int dm_alert_efmt_upload(dm_handle* h) {
    if (!h->fmt_set || !h->h_fmt || !h->d_afmt.get()) return DM_OK;
    std::unique_ptr<DmFormat> ef(new (std::nothrow) DmFormat);
    if (!ef) return dm_fail(DM_ERR_ARG, "out of host memory");
    dm_alert_efmt_build(*h->h_fmt, h->alert_time_cap, ef.get());
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess) e = dm_upload(h->d_efmt, *ef, h->last_stream);
    if (e == cudaSuccess) h->efmt_slots = ef->max_slots;
    if (e != cudaSuccess) return dm_fail(DM_ERR_CUDA, "encoder format: %s", cudaGetErrorString(e));
    return DM_OK;
}

extern "C" int dm_set_alert_format(dm_handle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* string_lens,
                                   const uint32_t* bits_off, const uint32_t* bits, uint32_t n_combos,
                                   const uint32_t* combo_off, const uint32_t* combo_members, uint32_t time_capture,
                                   uint64_t out_cap) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (!string_lens || (!strings && n_strings)) return dm_fail(DM_ERR_ARG, "strings missing");
    if (out_cap == 0) return dm_fail(DM_ERR_ARG, "out_cap must be positive");
    std::unique_ptr<DmAlertFmt> f(new (std::nothrow) DmAlertFmt);
    if (!f) return dm_fail(DM_ERR_ARG, "out of host memory");
    const char* why = dm_alert_fmt_build(h->h_keys, n_strings, strings, string_lens, bits_off, bits, n_combos, combo_off,
                                         combo_members, time_capture, f.get());
    if (why) return dm_fail(DM_ERR_ARG, "dm_set_alert_format: %s", why);
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->last_stream);
    if (e == cudaSuccess && !h->d_afmt.get()) {
        // everything the encoder needs, once: per record a rank, per anomaly-list entry a record's line, mask, offset and
        // size, the scan's tile sums.  Kept only when every allocation succeeded, so that a failed call leaves the
        // handle without an encoder (and a later call allocates again).
        DmDev<DmAlertFmt> d_afmt;
        DmDev<DmAlertHeader> d_ahdr;
        DmPinned<DmAlertHeader> h_ahdr;
        DmDev<uint8_t> d_alert;
        e = d_afmt.alloc(1);
        if (e == cudaSuccess) e = d_ahdr.alloc(1);
        if (e == cudaSuccess) e = h_ahdr.alloc(1);
        if (e == cudaSuccess) e = d_alert.alloc(dm_alert_scratch(nullptr, h->max_lines, h->anomaly_cap, nullptr, nullptr));
        if (e == cudaSuccess) {
            h->d_afmt = std::move(d_afmt); h->d_ahdr = std::move(d_ahdr); h->h_ahdr = std::move(h_ahdr); h->d_alert = std::move(d_alert);
        }
    }
    if (e == cudaSuccess && out_cap != h->d_aout.cap()) {
        h->d_aout.reset();
        e = h->d_aout.alloc(out_cap);
    }
    if (e == cudaSuccess) e = dm_upload(h->d_afmt, *f, h->last_stream);
    if (e != cudaSuccess) return dm_fail(DM_ERR_CUDA, "dm_set_alert_format: %s", cudaGetErrorString(e));
    h->alert_time_cap = time_capture < DM_FMT_MAX_CAPTURES ? time_capture : DMA_NONE;
    return dm_alert_efmt_upload(h);
}

template <typename T>
static void dm_alert_scan(T* d, uint64_t n, T* tile_sums, T* total, cudaStream_t st) {
    const uint32_t tiles = (uint32_t)std::max<uint64_t>(1, dm_alert_tiles(n));
    dm_k_alert_scan_tiles<T><<<tiles, DMA_THREADS, 0, st>>>(d, n, tile_sums);
    dm_k_alert_scan_top<T><<<1, DMA_THREADS, 0, st>>>(tile_sums, tiles, total);
    dm_k_alert_scan_apply<T><<<tiles, DMA_THREADS, 0, st>>>(d, n, tile_sums);
}

extern "C" int dm_encode_alerts(dm_handle* h, uint64_t first_log_id, int64_t first_alert_id, int64_t now, uint8_t* out,
                                uint64_t out_cap, uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    if (!h || !out_len || !n_alerts || !declined) return dm_fail(DM_ERR_ARG, "NULL argument");
    if (out_cap && !out) return dm_fail(DM_ERR_ARG, "out is NULL");
    if (!h->d_afmt.get() || !h->d_aout.get()) return dm_fail(DM_ERR_STATE, "dm_set_alert_format has not been called");
    if (h->last_src == DMA_SRC_NONE)
        return dm_fail(DM_ERR_STATE, "the last batch did not come from dm_process_lines, dm_process_logs, dm_process_records "
                                     "or dm_collect");
    *out_len = 0;
    *n_alerts = 0;
    *declined = 0;
    // A collected slot: its kernels have finished (dm_collect waited for them) and its header is the one dm_collect
    // read; dm_sync would put the handle's own header in its place.  The encoder runs on the slot's output stream, so
    // the other slot's kernels, in flight on the compute stream, keep running and their overlap chain stays intact.
    const bool from_slot = h->last_src == DMA_LINES && h->last_slot >= 0 && h->last_buf == h->slots[h->last_slot].d_in.get();
    const dm_handle::Slot* sl = from_slot ? &h->slots[h->last_slot] : nullptr;
    if (sl) {
        DM_CUDA(cudaSetDevice(h->device));
    } else {
        const int rc = dm_sync(h, nullptr, nullptr);
        if (rc != DM_OK) return rc;
    }
    const uint32_t src = h->last_src;
    uint64_t n_lines;
    bool over;
    const uint64_t n_flagged = dm_alert_entries(src, sl ? *sl->h_hdr.get() : *h->h_hdr.get(), h->last_n_records, h->anomaly_cap, &n_lines,
                                                &over);
    if (over) {
        *n_alerts = n_flagged;
        *declined = 1;
        return DM_OK;
    }
    if (n_flagged == 0) return DM_OK;
    const uint32_t entries = (uint32_t)n_flagged;
    cudaStream_t st = sl ? sl->st_out.get() : h->last_stream;
    dm_break_chain(h, st);
    DmAlertArgs a;
    unsigned long long* tile_sums;
    dm_alert_scratch((uint8_t*)h->d_alert.get(), h->max_lines, h->anomaly_cap, &a, &tile_sums);
    a.fmt = h->d_afmt.get(); a.buf = h->last_buf; a.nbytes = h->last_nbytes; a.scores = h->last_scores;
    a.anoms = sl ? sl->d_anoms.get() : h->d_anoms.get(); a.n_entries = entries; a.n_lines = n_lines;
    a.ahdr = h->d_ahdr.get(); a.first_log_id = first_log_id; a.first_alert_id = first_alert_id; a.now = now;
    a.out = h->d_aout.get(); a.out_cap = std::min<uint64_t>(out_cap, h->d_aout.cap());
    a.efmt = h->d_efmt.get(); a.nbuf = h->d_norm.get();
    a.src = src;
    if (src == DMA_LOGS) {
        float* rscores;
        uint8_t* rflags;
        const DmLogsArgs la = dm_logs_carve(h->d_logs.get(), h->logs_cap, h->logs_chunks, h->d_lhdr.get(), &rscores, &rflags);
        a.pay = h->d_in.get(); a.pay_off = la.rec_off; a.pay_len = la.rec_len;
        a.log_line = la.rec_line; a.log_dst = la.line_dst;
    } else if (src == DMA_RECORDS) {
        a.pay = h->d_in.get(); a.pay_off = h->d_vals.get(); a.pay_len = h->d_vals.get() + n_lines;
        a.scores = h->d_scores.get(); a.flags = h->d_flags.get(); a.masks = h->d_masks.get(); a.mons = h->d_mons.get();
    }
    bool fmtl;
    uint64_t mark_n;
    const DmAlertKernel k_mark = dm_alert_mark_kernel(src, false, n_lines, entries, &mark_n);
    const DmAlertKernel k_gather = dm_alert_mark_kernel(src, true, n_lines, entries, &mark_n);
    const DmAlertKernel k_size = dm_alert_pass_kernel(src, h->fmt_set, h->fmt_norm, false, &fmtl);
    const DmAlertKernel k_write = dm_alert_pass_kernel(src, h->fmt_set, h->fmt_norm, true, &fmtl);
    // log_format mode: the size and write passes re-run the matcher (one thread per record, DM_FMTL_THREADS per CTA)
    if (fmtl && !h->d_efmt.get()) return dm_fail(DM_ERR_STATE, "no log_format for the alert encoder");
    const unsigned mgrid = dm_grid(mark_n, DMA_THREADS, (uint64_t)h->sm_count * 8);
    const unsigned threads = fmtl ? DM_FMTL_THREADS : DMA_THREADS;
    const unsigned pgrid = dm_grid(entries, threads, (uint64_t)h->sm_count * (fmtl ? 32 : 8));
    const size_t smem = fmtl ? (size_t)2 * h->efmt_slots * DM_FMTL_THREADS * sizeof(uint2) : 0;
    DM_CUDA(cudaMemsetAsync(h->d_ahdr.get(), 0, sizeof(DmAlertHeader), st));
    DM_CUDA(cudaMemsetAsync(a.rank, 0, n_lines * 4, st));
    DM_CUDA(cudaMemsetAsync(a.rec_mask, 0, (uint64_t)entries * 4, st));
    k_mark<<<mgrid, DMA_THREADS, 0, st>>>(a);
    dm_alert_scan<uint32_t>(a.rank, n_lines, (uint32_t*)tile_sums, &h->d_ahdr.get()->n_alerts, st);
    k_gather<<<mgrid, DMA_THREADS, 0, st>>>(a);
    k_size<<<pgrid, threads, smem, st>>>(a);
    dm_alert_scan<unsigned long long>(a.size, entries, tile_sums, &h->d_ahdr.get()->total, st);
    k_write<<<pgrid, threads, smem, st>>>(a);
    h->launches += 10;
    DM_CUDA(cudaGetLastError());
    DM_CUDA(cudaMemcpyAsync(h->h_ahdr.get(), h->d_ahdr.get(), sizeof(DmAlertHeader), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    const DmAlertHeader ah = *h->h_ahdr.get();
    *n_alerts = ah.n_alerts;
    *out_len = ah.total;
    if (ah.declined || ah.total > a.out_cap) { *declined = 1; return DM_OK; }
    if (ah.total) DM_CUDA(cudaMemcpyAsync(out, h->d_aout.get(), ah.total, cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// pipelined host path
// ---------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------
// The MatcherParser stage: LogSchema records in, ParserSchemas out (dm_kernels_parse.cuh)
// ---------------------------------------------------------------------------------------
extern "C" int dm_set_parser_format(dm_handle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* string_lens,
                                    const uint32_t* capture_order) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (!h->fmt_set || !h->h_fmt) return dm_fail(DM_ERR_STATE, "dm_set_format has not been called");
    if (!string_lens || (!strings && n_strings)) return dm_fail(DM_ERR_ARG, "strings missing");
    std::unique_ptr<DmParseFmt> P(new (std::nothrow) DmParseFmt);
    std::unique_ptr<DmFormat> pf(new (std::nothrow) DmFormat);
    if (!P || !pf) return dm_fail(DM_ERR_ARG, "out of host memory");
    const char* why = dm_parse_fmt_build(*h->h_fmt, n_strings, strings, string_lens, capture_order, P.get());
    if (why) return dm_fail(DM_ERR_ARG, "dm_set_parser_format: %s", why);
    dm_parse_efmt_build(*h->h_fmt, pf.get());
    cudaError_t e = cudaSetDevice(h->device);
    if (e == cudaSuccess) e = h->h_ptotal.alloc(1);
    if (e == cudaSuccess) e = dm_upload(h->d_pf, *P, h->last_stream);
    if (e == cudaSuccess) e = dm_upload(h->d_pfmt, *pf, h->last_stream);
    if (e == cudaSuccess) h->pfmt_slots = pf->max_slots;
    if (e != cudaSuccess) return dm_fail(DM_ERR_CUDA, "dm_set_parser_format: %s", cudaGetErrorString(e));
    h->parse_set = true;
    return DM_OK;
}

extern "C" int dm_parse_logs(dm_handle* h, const uint8_t* buf, uint64_t nbytes, int delimited, int64_t first_parsed_id,
                             int64_t now, const uint8_t** out, uint64_t* out_len, uint64_t* n_records_out,
                             uint64_t* n_emitted_out, uint64_t* n_malformed_out) {
    if (!h || !out || !out_len) return dm_fail(DM_ERR_ARG, "NULL argument");
    if (nbytes && !buf) return dm_fail(DM_ERR_ARG, "buf is NULL");
    if (!h->parse_set) return dm_fail(DM_ERR_STATE, "dm_set_parser_format has not been called since the last dm_set_format");
    if (nbytes > h->max_batch_bytes) return dm_fail(DM_ERR_CAPACITY, "message of %llu bytes exceeds max_batch_bytes=%llu", (unsigned long long)nbytes, (unsigned long long)h->max_batch_bytes);
    *out = h->h_pout.get();
    *out_len = 0;
    DmFrames fr;
    int rc = dm_logs_frames(h, buf, nbytes, delimited, &fr);
    if (rc != DM_OK) return rc;
    const uint32_t n_records = (uint32_t)fr.off.size();
    h->last_src = DMA_SRC_NONE;                               // (d_in no longer holds the last detected batch)
    DmLogsArgs la;
    float* rscores;
    uint8_t* rflags;
    rc = dm_logs_unwrap(h, buf, nbytes, fr, 0, false, &la, &rscores, &rflags);
    if (rc != DM_OK) return rc;
    cudaStream_t st = h->stream.get();
    const uint64_t words = dm_parse_scratch(nullptr, n_records, nullptr, nullptr, nullptr);
    if (words > h->d_psize.cap()) {
        DM_CUDA(cudaStreamSynchronize(st));
        DM_CUDA(h->d_psize.grow(words, std::max<uint64_t>(2 * words, 8192)));
    }
    DmParseArgs a = dm_parse_args(la, h->d_pf.get(), h->d_pfmt.get(), h->d_norm.get(), first_parsed_id, now);
    unsigned long long *tile_sums, *d_total;
    dm_parse_scratch(h->d_psize.get(), n_records, &a, &tile_sums, &d_total);
    const bool norm = h->fmt_norm;
    if (norm && !h->d_norm.get()) return dm_fail(DM_ERR_STATE, "no R-norm scratch");
    const size_t smem = (size_t)2 * h->pfmt_slots * DM_FMTL_THREADS * sizeof(uint2);
    const unsigned grid = dm_grid(n_records, DM_FMTL_THREADS, (uint64_t)h->sm_count * 32);
    DM_CUDA(cudaMemsetAsync(d_total, 0, sizeof(unsigned long long), st));
    if (n_records) {
        dm_parse_kernel(norm, false)<<<grid, DM_FMTL_THREADS, smem, st>>>(a);
        dm_alert_scan<unsigned long long>(a.size, n_records, tile_sums, d_total, st);
        h->launches += 4;
        DM_CUDA(cudaGetLastError());
    }
    DM_CUDA(cudaMemcpyAsync(h->h_ptotal.get(), d_total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    const uint64_t total = *h->h_ptotal.get(), n_emitted = h->h_lhdr.get()->n_lines;
    const uint64_t cap = dm_grow_cap(h->d_pout.cap(), total);
    if (cap != h->d_pout.cap()) {                              // (both or neither: the old pair is freed first)
        *out = nullptr;
        h->d_pout.reset();
        h->h_pout.reset();
        DmDev<uint8_t> d_pout; DmPinned<uint8_t> h_pout;
        DM_CUDA(d_pout.alloc(cap));
        DM_CUDA(h_pout.alloc(cap));
        h->d_pout = std::move(d_pout);
        h->h_pout = std::move(h_pout);
    }
    if (total) {
        a.out = h->d_pout.get(); a.out_cap = h->d_pout.cap();
        dm_parse_kernel(norm, true)<<<grid, DM_FMTL_THREADS, smem, st>>>(a);
        h->launches++;
        DM_CUDA(cudaGetLastError());
        DM_CUDA(cudaMemcpyAsync(h->h_pout.get(), h->d_pout.get(), total, cudaMemcpyDeviceToHost, st));
        DM_CUDA(cudaStreamSynchronize(st));
    }
    *out = h->h_pout.get();
    *out_len = total;
    if (n_records_out) *n_records_out = n_records;
    if (n_emitted_out) *n_emitted_out = n_emitted;
    if (n_malformed_out) *n_malformed_out = n_records - n_emitted;
    return DM_OK;
}

static int dm_slots_init(dm_handle* h) {
    if (h->slots_ready) return DM_OK;
    DM_CUDA(h->st_in.create());
    for (auto& slot : h->slots) {
        dm_handle::Slot sl;                                    // (kept only when all of it was created)
        DM_CUDA(sl.d_in.alloc(h->max_batch_bytes + 256, true));
        DM_CUDA(sl.d_flags.alloc(h->max_lines + 16));
        DM_CUDA(sl.d_scores.alloc(h->max_lines + 4));
        DM_CUDA(sl.d_hdr.alloc(1, true));
        DM_CUDA(sl.d_anoms.alloc(h->anomaly_cap));
        DM_CUDA(sl.h_hdr.alloc(1));
        DM_CUDA(sl.h_flags.alloc(h->max_lines + 16));
        DM_CUDA(sl.h_scores.alloc(h->max_lines + 4));
        DM_CUDA(sl.ev_in.create());
        DM_CUDA(sl.ev_comp.create());
        DM_CUDA(sl.ev_hdr.create());
        DM_CUDA(sl.st_out.create());
        slot = std::move(sl);
    }
    h->slots_ready = true;
    return DM_OK;
}

extern "C" int dm_submit_lines(dm_handle* h, const uint8_t* host_buf, uint64_t nbytes, uint64_t n_train_lines, uint32_t slot) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (slot > 1) return dm_fail(DM_ERR_ARG, "slot must be 0 or 1");
    if (nbytes > h->max_batch_bytes)
        return dm_fail(DM_ERR_CAPACITY, "message of %llu bytes exceeds max_batch_bytes=%llu", (unsigned long long)nbytes, (unsigned long long)h->max_batch_bytes);
    if (nbytes && !host_buf) return dm_fail(DM_ERR_ARG, "host_buf is NULL");
    if (h->kernel_variant != 6) return dm_fail(DM_ERR_STATE, "the pipelined path runs the stream kernel (DM_KERNEL=lanes is set)");
    if (h->fmt_set) return dm_fail(DM_ERR_STATE, "the pipelined path tokenises key=value records; with a log_format use dm_process_lines");
    if (h->mons_set && h->h_mons.n_combos > 0) return dm_fail(DM_ERR_STATE, "combination monitors run in dm_process_lines / dm_process_records, not in the pipelined path");
    DM_CUDA(cudaSetDevice(h->device));
    int rc = dm_slots_init(h);
    if (rc != DM_OK) return rc;
    dm_handle::Slot& sl = h->slots[slot];
    if (sl.busy) return dm_fail(DM_ERR_STATE, "slot %u was submitted and not collected yet", slot);
    if (nbytes) DM_CUDA(cudaMemcpyAsync(sl.d_in.get(), host_buf, nbytes, cudaMemcpyHostToDevice, h->st_in.get()));
    DM_CUDA(cudaMemsetAsync(sl.d_in.get() + nbytes, 0, 64, h->st_in.get()));
    h->slot_nbytes[slot] = nbytes;
    DM_CUDA(cudaEventRecord(sl.ev_in.get(), h->st_in.get()));
    cudaStream_t st = h->stream.get();                       // ONE compute stream: submission order = processing order
    rc = dm_use_stream(h, st);
    if (rc != DM_OK) return rc;
    h->last_src = DMA_SRC_NONE;
    DM_CUDA(cudaStreamWaitEvent(st, sl.ev_in.get(), 0));
    if (nbytes == 0) DM_CUDA(cudaMemsetAsync(sl.d_hdr.get(), 0, sizeof(DmBatchHeader), st));
    const int launched = dmx_launch(&h->dmx, sl.d_in.get(), nbytes, n_train_lines, h->table, sl.d_flags.get(), sl.d_scores.get(), h->max_lines, sl.d_anoms.get(),
                                    h->anomaly_cap, sl.d_hdr.get(), h->d_stats.get(), h->max_lines, st, true, false, dm_prof_mark_cb, h);
    if (launched < 0) return dm_fail(DM_ERR_CUDA, "stream kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    h->launches += (uint64_t)launched;
    DM_CUDA(cudaEventRecord(sl.ev_comp.get(), st));
    DM_CUDA(cudaStreamWaitEvent(sl.st_out.get(), sl.ev_comp.get(), 0));
    DM_CUDA(cudaMemcpyAsync(sl.h_hdr.get(), sl.d_hdr.get(), sizeof(DmBatchHeader), cudaMemcpyDeviceToHost, sl.st_out.get()));
    DM_CUDA(cudaEventRecord(sl.ev_hdr.get(), sl.st_out.get()));
    sl.busy = true;
    return DM_OK;
}

extern "C" int dm_collect(dm_handle* h, uint32_t slot, const uint8_t** flags_out, const float** scores_out,
                          uint64_t* n_lines_out, uint64_t* n_anomalies_out) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (slot > 1 || !h->slots_ready || !h->slots[slot].busy) return dm_fail(DM_ERR_STATE, "slot %u has nothing to collect", slot);
    DM_CUDA(cudaSetDevice(h->device));
    dm_handle::Slot& sl = h->slots[slot];
    DM_CUDA(cudaEventSynchronize(sl.ev_hdr.get()));
    sl.busy = false;
    *h->h_hdr.get() = *sl.h_hdr.get();
    int rc = dm_check_device_errors(h);
    if (rc != DM_OK) return rc;
    const uint64_t n = sl.h_hdr.get()->n_lines;
    if (n && (flags_out || scores_out)) {
        if (flags_out) DM_CUDA(cudaMemcpyAsync(sl.h_flags.get(), sl.d_flags.get(), n, cudaMemcpyDeviceToHost, sl.st_out.get()));
        if (scores_out) DM_CUDA(cudaMemcpyAsync(sl.h_scores.get(), sl.d_scores.get(), n * sizeof(float), cudaMemcpyDeviceToHost, sl.st_out.get()));
        DM_CUDA(cudaStreamSynchronize(sl.st_out.get()));
    }
    if (flags_out) *flags_out = sl.h_flags.get();
    if (scores_out) *scores_out = sl.h_scores.get();
    if (n_lines_out) *n_lines_out = n;
    if (n_anomalies_out) *n_anomalies_out = sl.h_hdr.get()->n_anomalies;
    // the slot's batch is now the last batch, for dm_encode_alerts
    h->last_buf = sl.d_in.get();
    h->last_nbytes = h->slot_nbytes[slot];
    h->last_scores = sl.d_scores.get();
    h->last_src = DMA_LINES;
    h->last_slot = (int)slot;
    return DM_OK;
}

// Reads the anomaly list of a batch (total entries written, at most anomaly_cap of them kept) and merges it
// (dm_anomalies_merge): *n_out = the records, the first cap of them go to out.
static int dm_fetch_anomalies(dm_handle* h, const dm_anomaly_t* d_list, uint32_t total, dm_anomaly_t* out, uint32_t cap, uint32_t* n_out) {
    const uint32_t have = std::min(total, h->anomaly_cap);
    *n_out = 0;
    if (have == 0) return DM_OK;
    std::vector<dm_anomaly_t> tmp(have);
    DM_CUDA(cudaMemcpy(tmp.data(), d_list, (uint64_t)have * sizeof(dm_anomaly_t), cudaMemcpyDeviceToHost));
    const uint32_t m = dm_anomalies_merge(tmp.data(), have);
    *n_out = m;
    if (out && cap) memcpy(out, tmp.data(), (uint64_t)std::min(m, cap) * sizeof(dm_anomaly_t));
    return DM_OK;
}

extern "C" int dm_collect_anomalies(dm_handle* h, uint32_t slot, dm_anomaly_t* out, uint32_t cap, uint32_t* n_out) {
    if (!h || !n_out) return dm_fail(DM_ERR_ARG, "NULL argument");
    if (slot > 1 || !h->slots_ready) return dm_fail(DM_ERR_STATE, "slot %u was never used", slot);
    DM_CUDA(cudaSetDevice(h->device));
    dm_handle::Slot& sl = h->slots[slot];
    if (sl.busy) return dm_fail(DM_ERR_STATE, "slot %u is still in flight: dm_collect it first", slot);
    return dm_fetch_anomalies(h, sl.d_anoms.get(), sl.h_hdr.get()->anomaly_list_count, out, cap, n_out);
}

extern "C" int dm_sync(dm_handle* h, uint64_t* n_lines_out, uint64_t* n_anomalies_out) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(cudaStreamWaitEvent(h->last_stream, h->ev_import.get(), 0));     // the last window import, whatever its stream
    DM_CUDA(cudaMemcpyAsync(h->h_hdr.get(), h->d_hdr.get(), sizeof(DmBatchHeader), cudaMemcpyDeviceToHost, h->last_stream));
    int rc = dm_fetch_errors(h, h->last_stream);
    if (rc != DM_OK) return rc;
    DM_CUDA(cudaStreamSynchronize(h->last_stream));
    rc = dm_header_with_errors(h);
    if (rc != DM_OK) return rc;
    if (n_lines_out) *n_lines_out = h->h_hdr.get()->n_lines;
    if (n_anomalies_out) *n_anomalies_out = h->h_hdr.get()->n_anomalies;
    return DM_OK;
}

extern "C" int dm_get_anomalies(dm_handle* h, dm_anomaly_t* out, uint32_t cap, uint32_t* n_out) {
    if (!h || !n_out) return dm_fail(DM_ERR_ARG, "NULL argument");
    DM_CUDA(cudaSetDevice(h->device));
    int rc = dm_sync(h, nullptr, nullptr);
    if (rc != DM_OK) return rc;
    const uint32_t total = h->h_hdr.get()->anomaly_list_count;
    *n_out = std::min<uint64_t>(total, h->h_hdr.get()->n_anomalies ? h->h_hdr.get()->n_anomalies : total);
    if (!out || cap == 0 || std::min(total, h->anomaly_cap) == 0) return DM_OK;
    return dm_fetch_anomalies(h, h->d_anoms.get(), total, out, cap, n_out);
}

static void dm_words_to_stats(const unsigned long long* w, dm_stats_t* out) {
    out->lines = w[0]; out->train_lines = w[1]; out->detect_lines = w[2]; out->anomalies = w[3];
    out->score_sum = w[4]; out->bytes = w[5]; out->known_keys = w[6]; out->bad_records = w[7];
    for (int k = 0; k < DM_MAX_KEYS; ++k) out->unknown_per_key[k] = w[8 + k];
}

extern "C" int dm_get_stats(dm_handle* h, dm_stats_t* out) {
    if (!h || !out) return dm_fail(DM_ERR_ARG, "NULL argument");
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(cudaStreamSynchronize(h->last_stream));
    DM_CUDA(cudaMemcpy(h->h_stats.get(), h->d_stats.get(), DM_STATS_WORDS * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    dm_words_to_stats(h->h_stats.get(), out);
    unsigned long long cnt = 0;
    DM_CUDA(cudaMemcpy(&cnt, h->table.count, sizeof(cnt), cudaMemcpyDeviceToHost));
    out->known_keys = cnt;
    return DM_OK;
}

extern "C" int dm_get_global_stats(dm_handle* h, dm_stats_t* out) {
    if (!h || !out) return dm_fail(DM_ERR_ARG, "NULL argument");
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(cudaStreamWaitEvent(h->last_stream, h->ev_import.get(), 0));     // the last window import, whatever its stream
    DM_CUDA(cudaStreamSynchronize(h->last_stream));
    DM_CUDA(cudaMemcpy(h->h_stats.get(), h->d_stats_global, DM_STATS_WORDS * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    dm_words_to_stats(h->h_stats.get(), out);
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// known-set export / import / reset
// ---------------------------------------------------------------------------------------
// Every key of the table (own records, peers, dm_import_known), sorted on the device (dm_kernels_window.cuh): the
// count comes from the table's counter, so a count query (cap 0) copies 8 bytes back and launches nothing.
extern "C" int dm_export_known(dm_handle* h, uint64_t* keys_out, uint64_t cap, uint64_t* n_out) {
    if (!h || !n_out) return dm_fail(DM_ERR_ARG, "NULL argument");
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->last_stream;                    // behind everything the handle enqueued
    dm_break_chain(h, st);
    unsigned long long n = 0;
    DM_CUDA(cudaMemcpyAsync(&n, h->table.count, sizeof(n), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    *n_out = n;
    if (!keys_out || cap == 0 || n == 0) return DM_OK;
    // the scratch holds the load limit's slots/2 keys; only a table filled past its limit (its training reported
    // DM_ERR_TABLE_FULL) holds more, and then the scratch grows once to its count
    const uint64_t slots = (uint64_t)h->table.mask + 1;
    if (h->known.kcap < n) {                                   // (both or neither: the old pair is freed first)
        h->known = DmKnownScratch{};
        h->known_buf.reset();
        h->h_known_hist.reset();
        const uint64_t kcap = std::max<uint64_t>(n, slots / 2);
        DmDev<uint8_t> buf; DmPinned<unsigned int> hist;
        DM_CUDA(buf.alloc(dm_known_scratch(nullptr, kcap, nullptr)));
        DM_CUDA(hist.alloc(DMK_HIST_WORDS));
        h->known_buf = std::move(buf);
        h->h_known_hist = std::move(hist);
        dm_known_scratch(h->known_buf.get(), kcap, &h->known);
    }
    DmKnownScratch& s = h->known;
    DM_CUDA(cudaMemsetAsync(s.hist, 0, DMK_HIST_WORDS * sizeof(unsigned int), st));
    dm_k_known_compact<<<dm_grid(slots, DMK_TILE, 4 * (uint64_t)h->sm_count), DMK_THREADS, 0, st>>>(
        h->table.slots, slots, s.a, s.kcap, s.hist + DMK_PASSES * DMK_BINS);
    dm_k_known_digits<<<dm_grid(n, DMK_THREADS * 16, 2 * (uint64_t)h->sm_count), DMK_THREADS, 0, st>>>(s.a, n, s.hist);
    DM_CUDA(cudaGetLastError());
    DM_CUDA(cudaMemcpyAsync(h->h_known_hist.get(), s.hist, DMK_HIST_WORDS * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    if (h->h_known_hist.get()[DMK_PASSES * DMK_BINS] != n)
        return dm_fail(DM_ERR_STATE, "the table holds %u keys, its count says %llu", h->h_known_hist.get()[DMK_PASSES * DMK_BINS], n);
    uint32_t shifts[DMK_PASSES];
    const uint32_t n_passes = dm_known_passes(h->h_known_hist.get(), n, shifts);
    const uint32_t tiles = (uint32_t)dm_known_tiles(n);
    unsigned long long *src = s.a, *dst = s.b;
    for (uint32_t p = 0; p < n_passes; ++p) {
        dm_k_known_count<<<tiles, DMK_THREADS, 0, st>>>(src, n, shifts[p], s.counts);
        dm_alert_scan<uint32_t>(s.counts, (uint64_t)DMK_BINS * tiles, s.tile_sums, s.hist + DMK_PASSES * DMK_BINS + 1, st);
        dm_k_known_scatter<<<tiles, DMK_THREADS, 0, st>>>(src, n, shifts[p], s.counts, dst);
        std::swap(src, dst);
    }
    DM_CUDA(cudaGetLastError());
    DM_CUDA(cudaMemcpyAsync(keys_out, src, std::min<uint64_t>(n, cap) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    DM_CUDA(cudaStreamSynchronize(st));
    return DM_OK;
}

extern "C" int dm_import_known(dm_handle* h, const uint64_t* keys, uint64_t n) {
    if (!h || (n && !keys)) return dm_fail(DM_ERR_ARG, "NULL argument");
    if (n == 0) return DM_OK;
    DM_CUDA(cudaSetDevice(h->device));
    DmDev<unsigned long long> d_tmp;
    DM_CUDA(d_tmp.alloc(n));
    DM_CUDA(cudaMemcpy(d_tmp.get(), keys, n * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemsetAsync(h->d_hdr.get(), 0, sizeof(DmBatchHeader), h->last_stream));
    dm_break_chain(h, h->last_stream);
    h->last_src = DMA_SRC_NONE;
    dm_k_insert_keys<<<std::max(1, (int)std::min<uint64_t>((n + 255) / 256, 1024)), 256, 0, h->last_stream>>>(h->table, d_tmp.get(), n, &h->d_hdr.get()->error);
    DM_CUDA(cudaGetLastError());
    return dm_sync(h, nullptr, nullptr);
}

extern "C" int dm_reset(dm_handle* h) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    DM_CUDA(cudaSetDevice(h->device));
    // on last_stream, behind everything the handle enqueued: a memset on the legacy stream would not order against the
    // handle's non-blocking streams, and the next call's kernels could read the table before it is cleared
    cudaStream_t st = h->last_stream;
    dm_break_chain(h, st);
    DM_CUDA(cudaMemsetAsync(h->table.slots, 0, ((uint64_t)h->table.mask + 1) * sizeof(unsigned long long), st));
    DM_CUDA(cudaMemsetAsync(h->table.count, 0, 2 * sizeof(unsigned long long), st));
    DM_CUDA(cudaMemsetAsync(h->d_stats.get(), 0, 3 * DM_STATS_WORDS * sizeof(unsigned long long), st));
    DM_CUDA(cudaMemsetAsync(h->d_hdr.get(), 0, sizeof(DmBatchHeader), st));
    DM_CUDA(cudaStreamSynchronize(st));
    h->novel_exported = 0;
    h->novel_pending = 0;
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// multi-GPU window exchange (buffer layout and kernels: dm_kernels_window.cuh, with
// DM_WINDOW_KEYS keys per rank segment)
// ---------------------------------------------------------------------------------------
extern "C" uint64_t dm_window_words(dm_handle* h, uint32_t world, int with_keys) {
    (void)h;
    return dm_window_n_words(world, with_keys != 0, DM_WINDOW_KEYS);
}

extern "C" int dm_window_export(dm_handle* h, uint64_t* dev_buf, uint32_t rank, uint32_t world, int with_keys, void* stream_) {
    if (!h || !dev_buf || rank >= world) return dm_fail(DM_ERR_ARG, "bad window arguments");
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream.get();     // (not recorded as the compute stream)
    dm_break_chain(h, st);
    DmWindowKeys wk{h->novel_exported, h->novel_exported, 0};
    if (with_keys) {
        // the number of keys learnt so far is needed on the host to bound the segment
        unsigned long long cnt[2];
        DM_CUDA(cudaMemcpyAsync(cnt, h->table.count, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        DM_CUDA(cudaStreamSynchronize(st));
        // at most DM_WINDOW_KEYS keys travel per window; the rest goes with the next one (dm_window_pending_keys).
        // Failing here instead would leave the other ranks waiting in the all-reduce.
        wk = dm_window_keys(h->novel_exported, cnt[1], h->table.novel_cap, DM_WINDOW_KEYS);
        h->novel_pending = wk.pending;
    }
    const uint64_t n_words = dm_window_words(h, world, with_keys);
    const uint64_t seg_off = dm_window_n_words(rank, true, DM_WINDOW_KEYS);
    dm_k_window_export<<<std::max(1, (int)std::min<uint64_t>((n_words + 255) / 256, 2048)), 256, 0, st>>>(
        (unsigned long long*)dev_buf, n_words, h->d_stats.get(), h->d_stats_exported, h->table.novel, wk.from, wk.to, seg_off,
        DM_WINDOW_KEYS, with_keys);
    DM_CUDA(cudaGetLastError());
    h->novel_exported = wk.to;
    return DM_OK;
}

extern "C" int dm_window_pending_keys(dm_handle* h, uint64_t* n_out) {
    if (!h || !n_out) return dm_fail(DM_ERR_ARG, "NULL argument");
    *n_out = h->novel_pending;
    return DM_OK;
}

extern "C" int dm_window_import(dm_handle* h, const uint64_t* dev_buf, uint32_t rank, uint32_t world, int with_keys, void* stream_) {
    if (!h || !dev_buf || rank >= world) return dm_fail(DM_ERR_ARG, "bad window arguments");
    DM_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream.get();     // (not recorded as the compute stream)
    dm_break_chain(h, st);
    // errors go to the handle's accumulating error word, which no launch overwrites: the next dm_sync or synchronous
    // dm_process_lines reports them (the batch header's word is rewritten by the next detection launch)
    dm_k_window_import<<<with_keys ? 256 : 1, 256, 0, st>>>((const unsigned long long*)dev_buf, world, rank, DM_WINDOW_KEYS,
                                                          h->d_stats_global, h->table, &h->dmx.d_shared.get()->error, with_keys);
    DM_CUDA(cudaGetLastError());
    DM_CUDA(cudaEventRecord(h->ev_import.get(), st));     // dm_sync and dm_get_global_stats wait for it
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// The window exchange done natively: export -> ncclAllReduce(sum, uint64) -> import, all
// enqueued by ONE call (the torch.distributed route costs ~30 us of host time per window,
// which is what bounds the multi-GPU step).  NCCL is resolved at run time (dlopen of the
// libnccl.so.2 the process already has -- PyTorch's -- so there is no link-time dependency).
// ---------------------------------------------------------------------------------------
#include <dlfcn.h>
namespace {
struct DmNcclUniqueId { char internal[128]; };
typedef int (*fn_ncclGetUniqueId)(DmNcclUniqueId*);
typedef int (*fn_ncclCommInitRank)(void**, int, DmNcclUniqueId, int);
typedef int (*fn_ncclAllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*fn_ncclCommDestroy)(void*);
typedef const char* (*fn_ncclGetErrorString)(int);
struct DmNccl {
    void* lib = nullptr;
    fn_ncclGetUniqueId get_id = nullptr;
    fn_ncclCommInitRank init_rank = nullptr;
    fn_ncclAllReduce all_reduce = nullptr;
    fn_ncclCommDestroy destroy = nullptr;
    fn_ncclGetErrorString err = nullptr;
};
DmNccl g_nccl;
const int DM_NCCL_UINT64 = 5, DM_NCCL_SUM = 0;      // ncclUint64, ncclSum (stable across NCCL 2.x)

int dm_nccl_load() {
    if (g_nccl.lib) return DM_OK;
    const char* names[] = {getenv("DM_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    void* lib = nullptr;
    for (const char* n : names) {
        if (!n) continue;
        lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (lib) break;
    }
    if (!lib) return dm_fail(DM_ERR_STATE, "libnccl.so.2 not found (set DM_NCCL_LIB): %s", dlerror());
    g_nccl.get_id = (fn_ncclGetUniqueId)dlsym(lib, "ncclGetUniqueId");
    g_nccl.init_rank = (fn_ncclCommInitRank)dlsym(lib, "ncclCommInitRank");
    g_nccl.all_reduce = (fn_ncclAllReduce)dlsym(lib, "ncclAllReduce");
    g_nccl.destroy = (fn_ncclCommDestroy)dlsym(lib, "ncclCommDestroy");
    g_nccl.err = (fn_ncclGetErrorString)dlsym(lib, "ncclGetErrorString");
    if (!g_nccl.get_id || !g_nccl.init_rank || !g_nccl.all_reduce || !g_nccl.destroy || !g_nccl.err)
        return dm_fail(DM_ERR_STATE, "libnccl lacks an expected symbol");
    g_nccl.lib = lib;
    g_nccl_destroy_hook = [](void* c) { g_nccl.destroy(c); };
    return DM_OK;
}
}  // namespace

extern "C" int dm_nccl_unique_id(uint8_t* out128) {
    if (!out128) return dm_fail(DM_ERR_ARG, "NULL argument");
    int rc = dm_nccl_load();
    if (rc != DM_OK) return rc;
    DmNcclUniqueId id;
    const int r = g_nccl.get_id(&id);
    if (r != 0) return dm_fail(DM_ERR_CUDA, "ncclGetUniqueId: %s", g_nccl.err(r));
    memcpy(out128, &id, sizeof(id));
    return DM_OK;
}

extern "C" int dm_nccl_init(dm_handle* h, const uint8_t* ids, uint32_t n_comms, uint32_t rank, uint32_t world) {
    if (!h || !ids || world == 0 || rank >= world || n_comms < 1 || n_comms > 2) return dm_fail(DM_ERR_ARG, "bad arguments");
    if (h->nccl_n) return dm_fail(DM_ERR_STATE, "the handle already has its communicators");
    int rc = dm_nccl_load();
    if (rc != DM_OK) return rc;
    DM_CUDA(cudaSetDevice(h->device));
    for (uint32_t k = 0; k < n_comms; ++k) {
        DmNcclUniqueId id;
        memcpy(&id, ids + 128 * k, sizeof(id));
        void* comm = nullptr;
        const int r = g_nccl.init_rank(&comm, (int)world, id, (int)rank);
        if (r != 0) return dm_fail(DM_ERR_CUDA, "ncclCommInitRank: %s", g_nccl.err(r));
        h->nccl_comm[k] = comm;
        DM_CUDA(h->d_win[k].alloc(dm_window_words(h, world, 1)));
        DM_CUDA(h->ev_win_done[k].create());
    }
    h->nccl_n = n_comms; h->nccl_rank = rank; h->nccl_world = world;
    return DM_OK;
}

extern "C" int dm_window_allreduce(dm_handle* h, int with_keys, void* stream_) {
    if (!h) return dm_fail(DM_ERR_ARG, "handle is NULL");
    if (!h->nccl_n) return dm_fail(DM_ERR_STATE, "dm_nccl_init has not been called");
    // consecutive windows alternate between the communicators (and their buffers): called on
    // alternating streams, two all-reduces are in flight, which matters at 8 ranks where one
    // export + all-reduce + import chain is longer than a step
    const uint32_t k = (uint32_t)(h->win_seq++ % h->nccl_n);
    cudaStream_t st = stream_ ? (cudaStream_t)stream_ : h->stream.get();     // (not recorded as the compute stream)
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(cudaStreamWaitEvent(st, h->ev_win_done[k].get(), 0));           // the buffer's previous window is through
    int rc = dm_window_export(h, (uint64_t*)h->d_win[k].get(), h->nccl_rank, h->nccl_world, with_keys, stream_);
    if (rc != DM_OK) return rc;
    const int r = g_nccl.all_reduce(h->d_win[k].get(), h->d_win[k].get(), (size_t)dm_window_words(h, h->nccl_world, with_keys),
                                    DM_NCCL_UINT64, DM_NCCL_SUM, h->nccl_comm[k], st);
    if (r != 0) return dm_fail(DM_ERR_CUDA, "ncclAllReduce: %s", g_nccl.err(r));
    rc = dm_window_import(h, (const uint64_t*)h->d_win[k].get(), h->nccl_rank, h->nccl_world, with_keys, stream_);
    if (rc != DM_OK) return rc;
    DM_CUDA(cudaEventRecord(h->ev_win_done[k].get(), st));
    return DM_OK;
}

// ---------------------------------------------------------------------------------------
// Host utility: write a host buffer back and evict it from the CPU caches.  A pinned buffer
// the CPU has just written sits in its caches as dirty lines, and the GPU's DMA reads of such
// lines are snooped out of the caches at a fraction of the DRAM streaming rate (measured:
// 16 MiB in 500-1500 us instead of 313 us, scripts/pinned_numa_diag.py).  bench.py flushes its
// pinned inputs once after filling them so that the end-to-end number does not depend on
// what the set-up code left in the L3.
// ---------------------------------------------------------------------------------------
#if defined(__x86_64__)
#include <emmintrin.h>
extern "C" int dm_host_cache_flush(const void* p, uint64_t nbytes) {
    if (!p && nbytes) return dm_fail(DM_ERR_ARG, "NULL argument");
    const char* c = (const char*)((uintptr_t)p & ~(uintptr_t)63);
    const char* e = (const char*)p + nbytes;
    _mm_mfence();
    for (; c < e; c += 64) _mm_clflush(c);
    _mm_mfence();
    return DM_OK;
}
#else
extern "C" int dm_host_cache_flush(const void* p, uint64_t nbytes) { (void)p; (void)nbytes; return DM_OK; }
#endif
