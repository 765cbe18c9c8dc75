// dm_kernels_index.cuh -- K_A, the row / record index of a message (sm_90a).
//
// dm_k_rowindex streams the message once (16-byte loads), counts the '\n' of every 512-byte row,
// turns the counts into a global exclusive prefix (tiles of 64 rows, decoupled look-back with
// 128-wide windows), zero-fills flags / scores, writes the batch header and, for the
// one-thread-per-record kernels (dm_kernels_lanes.cuh, dm_kernels_format.cuh), the first byte of
// every record (line_start[]).  The default key=value path (dm_kernels_stream.cuh) does not need it.
// Also here: programmatic-dependent-launch helpers shared by all kernels.
#pragma once
#include "dm_device.cuh"

#define DMR_ROW 512u
#define DMR_TILE_ROWS 64u
#define DMR_A_THREADS 256
#define DMR_GROUP 2u          // rows fetched per atomic (after the static share)

struct DmRowsArgs {
    const uint8_t* buf;
    uint64_t nbytes;
    uint32_t n_rows;
    uint32_t n_tiles;
    uint32_t* row_prefix;             // n_rows entries
    unsigned long long* tile_state;   // look-back words of K_A
    uint32_t epoch;
    const DmKeys* keys;
    DmTable table;
    uint8_t* flags;
    float* scores;
    uint64_t out_cap;
    dm_anomaly_t* anomalies;
    uint32_t anomaly_cap;
    DmBatchHeader* hdr;
    unsigned long long* stats;
    unsigned long long* row_ctr;      // monotonically increasing across launches
    unsigned long long ctr_base;
    uint64_t line_lo, line_hi;        // K_B handles records with index in [lo, hi)
    uint64_t n_train_lines;
    uint64_t max_lines;
    unsigned int* aux_counts;         // staged variant: list counters cleared by K_A (else NULL)
    uint32_t group;                   // rows fetched per atomic by a K_B warp
    uint32_t static_rows;             // rows every K_B warp takes without asking (warp w: rows [w*S, (w+1)*S))
    unsigned long long* timeline;     // diagnostics (DM_ROWS_TIMELINE): per K_B warp {smid, t_first, t_work_end, t_exit} in ns, else NULL
    uint32_t* line_start;             // lanes variant: K_A also writes the record index (else NULL):
                                      // line_start[g] = first byte of record g, line_start[n] = end sentinel
};

// Programmatic dependent launch (PDL).  The two kernels of a step and the first kernel of the
// next step are launched with cudaLaunchAttributeProgrammaticStreamSerialization: a kernel may
// be scheduled while its predecessor in the stream is still running, does whatever does not
// depend on it (K_B: key tables to shared memory; K_A: stream the rows in and count), and calls
// dm_pdl_wait() before it touches anything the predecessor reads or writes.  Launched without the
// attribute both calls are no-ops.
__device__ __forceinline__ void dm_pdl_wait() {
#ifndef DM_EMU
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
__device__ __forceinline__ void dm_pdl_launch_dependents() {
#ifndef DM_EMU
    asm volatile("griddepcontrol.launch_dependents;");
#endif
}

// 16-bit '\n' mask of this lane's chunk of a row, slack bytes behind the message dropped
__device__ __forceinline__ uint32_t dm_row_nl_mask(const uint4& v, uint64_t off, uint64_t nbytes) {
    const uint32_t f0 = dm_eqflags(v.x, 0x0A0A0A0Au), f1 = dm_eqflags(v.y, 0x0A0A0A0Au);
    const uint32_t f2 = dm_eqflags(v.z, 0x0A0A0A0Au), f3 = dm_eqflags(v.w, 0x0A0A0A0Au);
    if ((f0 | f1 | f2 | f3) == 0) return 0;
    uint32_t m = dm_flags_to_nib(f0) | (dm_flags_to_nib(f1) << 4) | (dm_flags_to_nib(f2) << 8) | (dm_flags_to_nib(f3) << 12);
    if (off + 16 > nbytes) m &= (1u << (uint32_t)(nbytes - off)) - 1u;
    return m;
}

// ---------------------------------------------------------------------------------------
// K_A: row index
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DMR_A_THREADS) dm_k_rowindex(DmRowsArgs a) {
    __shared__ uint32_t s_rowcnt[DMR_TILE_ROWS];
    __shared__ uint32_t s_rowpre[DMR_TILE_ROWS];      // '\n' in front of each row, inside the tile
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_total;
    const uint8_t* __restrict__ buf = a.buf;
    const uint64_t nbytes = a.nbytes;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t tile = blockIdx.x;

    dm_pdl_launch_dependents();                       // the detect kernel of this step may be scheduled now
    // newline count of each row of the tile: 8 warps x 8 rows, all 8 loads of a warp in flight
    uint32_t nlm[8];                                  // this lane's '\n' masks (kept for the record index)
    {
        const uint32_t rr = warp * 8;
        uint4 v[8];
        uint64_t off[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            off[i] = ((uint64_t)tile * DMR_TILE_ROWS + rr + i) * DMR_ROW + (uint64_t)lane * 16;
            v[i] = make_uint4(0, 0, 0, 0);
            if (off[i] < nbytes) v[i] = __ldg(reinterpret_cast<const uint4*>(buf + off[i]));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t m = off[i] < nbytes ? dm_row_nl_mask(v[i], off[i], nbytes) : 0u;
            nlm[i] = m;
            const uint32_t c = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(m));
            if (lane == 0) s_rowcnt[rr + i] = c;
        }
    }
    // Everything up to and including the look-back below only reads the message and touches
    // tile_state, which no other kernel uses (epoch-tagged): under PDL it runs while the previous
    // step's detect kernel is still busy.  dm_pdl_wait() comes right before the first write to
    // anything that kernel reads or writes (row_prefix, header, outputs).
    __syncthreads();

    if (warp == 0) {
        // exclusive prefix of the 64 row counts (2 per lane), then the tile's global base
        uint32_t c[2], lane_sum = 0;
#pragma unroll
        for (int i = 0; i < 2; ++i) { c[i] = s_rowcnt[lane * 2 + i]; lane_sum += c[i]; }
        uint32_t incl = lane_sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
            if ((int)lane >= d) incl += y;
        }
        const uint32_t agg = __shfl_sync(0xffffffffu, incl, 31);
        const unsigned long long tag = (unsigned long long)a.epoch << 34;
        unsigned long long excl = 0;
        if (tile > 0) {
            if (lane == 0) atomicExch(a.tile_state + tile, tag | (DMT_ST_AGG << 32) | agg);
            long long hi = (long long)tile - 1;
            bool done = false;
            while (!done) {
                unsigned long long st[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const long long idx = hi - 32 * j - (long long)lane;
                    st[j] = idx >= 0 ? *((volatile unsigned long long*)(a.tile_state + idx)) : 0ull;
                }
                int consumed = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (done || consumed < j) continue;
                    const long long idx = hi - 32 * j - (long long)lane;
                    unsigned long long w = st[j];
                    if (idx >= 0 && (w >> 34) != a.epoch) w = 0;
                    const uint32_t status = idx >= 0 ? (uint32_t)((w >> 32) & 3u) : (uint32_t)DMT_ST_PREFIX;
                    const uint32_t not_ready = __ballot_sync(0xffffffffu, status == 0);
                    const uint32_t is_pref = __ballot_sync(0xffffffffu, status == DMT_ST_PREFIX);
                    const uint32_t first_pref = is_pref ? (uint32_t)(__ffs(is_pref) - 1) : 32u;
                    const uint32_t upto = first_pref < 32u ? first_pref : 31u;
                    const uint32_t win = upto == 31u ? 0xffffffffu : ((2u << upto) - 1u);
                    if (not_ready & win) continue;
                    const uint32_t val = (lane <= upto && idx >= 0) ? (uint32_t)w : 0u;
                    excl += __reduce_add_sync(0xffffffffu, val);
                    consumed = j + 1;
                    if (first_pref < 32u) done = true;
                }
                hi -= 32 * consumed;
                if (!done && consumed < 4) __nanosleep(20);
            }
        }
        if (lane == 0) atomicExch(a.tile_state + tile, tag | (DMT_ST_PREFIX << 32) | (unsigned long long)((uint32_t)excl + agg));
        dm_pdl_wait();
        uint32_t run = (uint32_t)excl + (incl - lane_sum);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const uint32_t row = tile * DMR_TILE_ROWS + lane * 2 + i;
            if (row < a.n_rows) a.row_prefix[row] = run;
            s_rowpre[lane * 2 + i] = run - (uint32_t)excl;
            run += c[i];
        }
        if (lane == 0) { s_base = excl; s_total = agg; }
        if (tile == a.n_tiles - 1 && lane == 0) {
            const unsigned long long nl = excl + agg;
            const bool tail = nbytes > 0 && buf[nbytes - 1] != 0x0Au;
            unsigned long long n_lines = nl + (tail ? 1ull : 0ull);
            // the last tile (the only one that knows the totals) initialises the whole batch header
            a.hdr->n_anomalies = 0; a.hdr->anomaly_list_count = 0;
            a.hdr->error = (n_lines > a.max_lines || n_lines > a.out_cap) ? DM_DEVERR_TOO_MANY_LINES : 0u;
            a.hdr->n_newlines = nl;
            a.hdr->n_lines = n_lines;
            if (a.aux_counts) { a.aux_counts[0] = 0; a.aux_counts[1] = 0; a.aux_counts[2] = 0; }
            const unsigned long long tr = a.n_train_lines < n_lines ? a.n_train_lines : n_lines;
            a.stats[0] += n_lines;
            a.stats[1] += tr;
            a.stats[2] += n_lines - tr;
            a.stats[5] += nbytes;
            if (tail) s_total = agg + 1;            // the unterminated last record is zero-filled here too
        }
    }
    __syncthreads();
    dm_pdl_wait();                                    // (warp 0 has waited already; the other warps write below)
    const unsigned long long base = s_base;
    if (a.line_start) {
        // lanes variant: the record index.  The '\n' at byte x with k '\n' in front of it ends
        // record k, so record k+1 starts at x+1.  (Every record's outputs are written by its own
        // lane there, no zero-fill.)
        if (tile == 0 && threadIdx.x == 0) a.line_start[0] = 0;
        if (tile == a.n_tiles - 1 && threadIdx.x == 0 && nbytes > 0 && buf[nbytes - 1] != 0x0Au) {
            const unsigned long long n_lines = base + s_total;          // s_total counts the unterminated record
            if (n_lines <= a.max_lines) a.line_start[n_lines] = (uint32_t)(nbytes + 1);
        }
        const uint32_t rr = warp * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t m = nlm[i];
            // records in front of this lane's chunk: tile base + row prefix + lower lanes of the row
            uint32_t incl = (uint32_t)__popc(m);
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
                if ((int)lane >= d) incl += y;
            }
            unsigned long long k = base + s_rowpre[rr + i] + (incl - (uint32_t)__popc(m));
            const uint64_t off = ((uint64_t)tile * DMR_TILE_ROWS + rr + i) * DMR_ROW + (uint64_t)lane * 16;
            while (m) {
                const uint32_t b = (uint32_t)__ffs(m) - 1u;
                m &= m - 1;
                ++k;
                if (k <= a.max_lines) a.line_start[k] = (uint32_t)(off + b + 1);
            }
        }
        return;
    }
    // zero-fill the outputs of the records that end in this tile
    const uint32_t total = s_total;
    for (uint32_t i = threadIdx.x; i < total; i += DMR_A_THREADS) {
        const unsigned long long g = base + i;
        if (g < a.out_cap) { a.flags[g] = 0; a.scores[g] = 0.0f; }
    }
}

// K_A's arguments for one message, writing the record index to line_start.  The look-back tag *epoch advances when
// the message has rows (else nothing is launched).  The fields dm_k_rowindex does not read stay zero.
static inline DmRowsArgs dm_rows_args(const uint8_t* buf, uint64_t nbytes, uint32_t* row_prefix, unsigned long long* tile_state,
                                      uint32_t* epoch, uint32_t* line_start, uint8_t* flags, float* scores, uint64_t out_cap,
                                      DmBatchHeader* hdr, unsigned long long* stats, uint64_t n_train_lines, uint64_t max_lines) {
    DmRowsArgs a{};
    a.buf = buf; a.nbytes = nbytes;
    a.n_rows = (uint32_t)((nbytes + DMR_ROW - 1) / DMR_ROW);
    a.n_tiles = (a.n_rows + DMR_TILE_ROWS - 1) / DMR_TILE_ROWS;
    a.row_prefix = row_prefix; a.tile_state = tile_state;
    if (a.n_rows) *epoch = (*epoch % 0x3FFFFFFEu) + 1u;
    a.epoch = *epoch;
    a.line_start = line_start; a.flags = flags; a.scores = scores; a.out_cap = out_cap;
    a.hdr = hdr; a.stats = stats; a.n_train_lines = n_train_lines; a.max_lines = max_lines;
    return a;
}

#ifndef DM_EMU
// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct DmRowsScratch {
    uint32_t* d_row_prefix = nullptr;
    unsigned long long* d_tile_state = nullptr;
    uint64_t max_rows = 0, max_tiles = 0;
    uint32_t epoch = 0;
    // K_A reads the message before it waits for its predecessor (programmatic dependent launch); a caller may have
    // produced that message with a kernel of its own on the same stream, so K_A is launched as an ordinary kernel
    bool pdl = false;
};

static inline int dm_rows_scratch_create(DmRowsScratch* s, uint64_t max_batch_bytes, int sm_count) {
    (void)sm_count;
    s->max_rows = (max_batch_bytes + DMR_ROW - 1) / DMR_ROW + 1;
    s->max_tiles = (s->max_rows + DMR_TILE_ROWS - 1) / DMR_TILE_ROWS + 1;
    if (cudaMalloc(&s->d_row_prefix, s->max_rows * sizeof(uint32_t)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMalloc(&s->d_tile_state, s->max_tiles * sizeof(unsigned long long)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMemset(s->d_tile_state, 0, s->max_tiles * sizeof(unsigned long long)) != cudaSuccess) return DM_ERR_CUDA;
    return DM_OK;
}

static inline void dm_rows_scratch_destroy(DmRowsScratch* s) {
    cudaFree(s->d_row_prefix);
    cudaFree(s->d_tile_state);
    s->d_row_prefix = nullptr; s->d_tile_state = nullptr;
}

// <<<>>> with the programmatic-stream-serialization attribute (see dm_pdl_wait)
template <typename... Args>
static inline void dm_launch_pdl_smem(void (*kernel)(Args...), unsigned grid, unsigned block, size_t smem, cudaStream_t st,
                                      bool pdl, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid, 1, 1); cfg.blockDim = dim3(block, 1, 1); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, args...);
}
template <typename Arg>
static inline void dm_launch_pdl(void (*kernel)(Arg), unsigned grid, unsigned block, cudaStream_t st, bool pdl, Arg arg) {
    dm_launch_pdl_smem(kernel, grid, block, 0, st, pdl, arg);
}

#endif  // DM_EMU
