// emu_known.cpp -- dm_export_known's kernels (dm_kernels_window.cuh) on the CPU emulator.  TEST INFRASTRUCTURE ONLY:
// built by tests/test_emu_known_export.py into tests/emu/_build/; never part of libdmdetect.so.
//
// An emulated known-set table (the slots, the counters and the novel list of a DmTable) filled by dm_k_insert_keys, as
// dm_import_known fills it, and exported with the launches dm_export_known enqueues: the same scratch layout
// (dm_known_scratch), pass plan (dm_known_passes) and per-tile grids.  The compaction and histogram kernels run on 2
// CTAs so that they take their stride loops; the scratch starts out hostile.
#include "cuda_emu.h"

#include <algorithm>
#include <vector>

#include "dm_kernels_window.cuh"

thread_local emu_dim3 threadIdx;
thread_local emu_dim3 blockIdx;
emu_dim3 blockDim, gridDim;
EmuBlock* g_emu_block = nullptr;
std::atomic<int> g_emu_or_flag[2];
std::vector<uint8_t> g_emu_dyn_smem;

// the blocks of a grid one after the other, one OS thread per CUDA thread
static void emu_launch_grid(unsigned blocks, unsigned threads, const std::function<void()>& body) {
    blockDim.x = threads;
    gridDim.x = blocks;
    for (unsigned b = 0; b < blocks; ++b) {
        EmuBlock blk;
        blk.warps = std::vector<EmuWarp>(threads / 32);
        g_emu_block = &blk;
        std::vector<std::thread> ts;
        ts.reserve(threads);
        for (unsigned t = 0; t < threads; ++t)
            ts.emplace_back([t, b, &body] {
                threadIdx.x = t;
                blockIdx.x = b;
                body();
            });
        for (auto& t : ts) t.join();
        g_emu_block = nullptr;
    }
}

void emu_launch(unsigned threads, const std::function<void()>& body) { emu_launch_grid(1, threads, body); }

struct EmuKnown {
    std::vector<unsigned long long> slots, novel;
    unsigned long long counts[2] = {0, 0};
    DmTable t;
};

extern "C" EmuKnown* emu_known_create(uint32_t log2) {
    EmuKnown* k = new EmuKnown();
    const uint64_t cap = 1ull << log2;
    k->slots.assign(cap, 0);
    k->novel.assign(cap / 2, 0);
    k->t.slots = k->slots.data();
    k->t.mask = (uint32_t)(cap - 1);
    k->t.limit = (uint32_t)(cap / 2);
    k->t.count = &k->counts[0];
    k->t.novel = k->novel.data();
    k->t.novel_count = &k->counts[1];
    k->t.novel_cap = (uint32_t)(cap / 2);
    return k;
}

extern "C" void emu_known_destroy(EmuKnown* k) { delete k; }

// as dm_import_known (dm_k_insert_keys on 2 CTAs of 32 threads); the DM_DEVERR_* bits
extern "C" uint32_t emu_known_insert(EmuKnown* k, const unsigned long long* keys, uint64_t n) {
    unsigned int err = 0;
    if (n) emu_launch_grid(2, 32, [&] { dm_k_insert_keys(k->t, keys, n, &err); });
    return err;
}

// the table's counter, which dm_export_known reads first
extern "C" uint64_t emu_known_count(EmuKnown* k) { return k->counts[0]; }

// As dm_export_known: at most cap keys of the table, ascending, to out; their count (all of them), or ~0 when the
// compaction counts another number of keys than the table's counter.  *n_passes: the radix passes run.
extern "C" uint64_t emu_known_export(EmuKnown* k, unsigned long long* out, uint64_t cap, uint32_t* n_passes) {
    const uint64_t n = k->counts[0], slots = k->slots.size();
    *n_passes = 0;
    if (!out || cap == 0 || n == 0) return n;
    DmKnownScratch s;
    const uint64_t kcap = std::max<uint64_t>(n, slots / 2);
    std::vector<unsigned long long> buf((dm_known_scratch(nullptr, kcap, nullptr) + 7) / 8, 0xDEADBEEFDEADBEEFull);
    dm_known_scratch(buf.data(), kcap, &s);
    memset(s.hist, 0, DMK_HIST_WORDS * sizeof(unsigned int));              // as the library's cudaMemsetAsync
    emu_launch_grid(dm_grid(slots, DMK_TILE, 2), DMK_THREADS, [&] {
        dm_k_known_compact(k->slots.data(), slots, s.a, s.kcap, s.hist + DMK_PASSES * DMK_BINS);
    });
    emu_launch_grid(dm_grid(n, DMK_THREADS, 2), DMK_THREADS, [&] { dm_k_known_digits(s.a, n, s.hist); });
    if (s.hist[DMK_PASSES * DMK_BINS] != n) return ~0ull;
    uint32_t shifts[DMK_PASSES];
    const uint32_t np = dm_known_passes(s.hist, n, shifts);
    const uint32_t tiles = (uint32_t)dm_known_tiles(n);
    const uint64_t n_counts = (uint64_t)DMK_BINS * tiles;
    const uint32_t scan_tiles = (uint32_t)std::max<uint64_t>(1, dm_alert_tiles(n_counts));
    unsigned int* total = s.hist + DMK_PASSES * DMK_BINS + 1;
    unsigned long long *src = s.a, *dst = s.b;
    for (uint32_t p = 0; p < np; ++p) {
        emu_launch_grid(tiles, DMK_THREADS, [&] { dm_k_known_count(src, n, shifts[p], s.counts); });
        // the library's dm_alert_scan<uint32_t>: tile sums, one CTA over them, tiles again
        emu_launch_grid(scan_tiles, DMA_THREADS, [&] { dm_k_alert_scan_tiles<uint32_t>(s.counts, n_counts, s.tile_sums); });
        emu_launch(DMA_THREADS, [&] { dm_k_alert_scan_top<uint32_t>(s.tile_sums, scan_tiles, total); });
        emu_launch_grid(scan_tiles, DMA_THREADS, [&] { dm_k_alert_scan_apply<uint32_t>(s.counts, n_counts, s.tile_sums); });
        emu_launch_grid(tiles, DMK_THREADS, [&] { dm_k_known_scatter(src, n, shifts[p], s.counts, dst); });
        std::swap(src, dst);
    }
    *n_passes = np;
    memcpy(out, src, std::min<uint64_t>(n, cap) * sizeof(unsigned long long));
    return n;
}
