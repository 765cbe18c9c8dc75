"""The owners of libdmdetect's CUDA runtime objects (csrc/dm_buf.h), on the CPU.

A small C++ program includes dm_buf.h against the CUDA toolkit's headers and links its own cudaMalloc / cudaHostAlloc /
cudaFree / cudaFreeHost (and event / stream create and destroy) instead of libcudart: they count live allocations,
catch a free of anything not live, and can fail the k-th allocation.  That is how every failure path of the owners
runs here, which a GPU cannot be made to do on purpose.
"""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "detectmateservice_b200", "csrc")

PROGRAM = r"""
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <string>
#include "dm_buf.h"

static std::set<void*> g_live;
static int g_allocs = 0, g_frees = 0, g_fail_at = -1, g_bad = 0;

static cudaError_t fake_alloc(void** p, size_t n) {
    if (++g_allocs == g_fail_at) return cudaErrorMemoryAllocation;
    *p = malloc(n ? n : 1);
    memset(*p, 0xAB, n);
    g_live.insert(*p);
    return cudaSuccess;
}
static cudaError_t fake_free(void* p) {
    ++g_frees;
    if (!p || !g_live.erase(p)) { ++g_bad; return cudaErrorInvalidValue; }
    free(p);
    return cudaSuccess;
}
extern "C" {
cudaError_t cudaMalloc(void** p, size_t n) { return fake_alloc(p, n); }
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned int) { return fake_alloc(p, n); }
cudaError_t cudaFree(void* p) { return fake_free(p); }
cudaError_t cudaFreeHost(void* p) { return fake_free(p); }
cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned int) { return fake_alloc((void**)e, 8); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { return fake_free((void*)e); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned int) { return fake_alloc((void**)s, 8); }
cudaError_t cudaStreamDestroy(cudaStream_t s) { return fake_free((void*)s); }
}

static int g_failed = 0;
#define CHECK(c) do { if (!(c)) { printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_failed; } } while (0)
static size_t live() { return g_live.size(); }

static void grow_within_capacity() {
    DmDev<int> b;
    CHECK(b.grow(10, 100) == cudaSuccess && b.cap() == 100 && g_allocs == 1);
    int* p = b.get();
    CHECK(b.grow(100, 400) == cudaSuccess && b.grow(1, 1) == cudaSuccess && b.alloc(64) == cudaSuccess);
    CHECK(g_allocs == 1 && g_frees == 0 && b.get() == p && b.cap() == 100);
    DmPinned<int> z;
    CHECK(z.alloc(5, true) == cudaSuccess);
    for (int i = 0; i < 5; ++i) CHECK(z.get()[i] == 0);
}

static void growth_frees_old_once() {
    DmDev<double> b;
    CHECK(b.alloc(10) == cudaSuccess);
    CHECK(b.grow(11, 40) == cudaSuccess && b.cap() == 40 && g_frees == 1 && live() == 1);
    g_fail_at = g_allocs + 1;
    CHECK(b.grow(41, 80) == cudaErrorMemoryAllocation);
    CHECK(b.get() == nullptr && b.cap() == 0 && live() == 0 && g_frees == 2);
    CHECK(b.grow(1, 8) == cudaSuccess && b.cap() == 8 && live() == 1);  // an empty owner allocates again
    b.reset();
    b.reset();
    CHECK(b.get() == nullptr && b.cap() == 0 && live() == 0 && g_frees == 3);
}

static void move_transfers() {
    DmPinned<char> a;
    CHECK(a.alloc(16) == cudaSuccess);
    char* p = a.get();
    DmPinned<char> b(std::move(a));
    CHECK(a.get() == nullptr && a.cap() == 0 && b.get() == p && b.cap() == 16 && g_frees == 0);
    DmPinned<char> c;
    CHECK(c.alloc(4) == cudaSuccess);
    c = std::move(b);                                     // frees what c held, once
    CHECK(b.get() == nullptr && b.cap() == 0 && c.get() == p && c.cap() == 16 && g_frees == 1 && live() == 1);
    DmEvent e1, e2;
    CHECK(e1.create() == cudaSuccess && e1.get() != nullptr);
    cudaEvent_t ev = e1.get();
    e2 = std::move(e1);
    CHECK(e1.get() == nullptr && e2.get() == ev && live() == 2);
}

struct Target { DmDev<char> d; DmPinned<int> h; DmDev<long> t; };

// Allocated into locals, moved into tg only when all three succeeded.
static cudaError_t fill(Target& tg, size_t n) {
    DmDev<char> d; DmPinned<int> h; DmDev<long> t;
    cudaError_t e = d.alloc(n);
    if (e == cudaSuccess) e = h.alloc(n);
    if (e == cudaSuccess) e = t.alloc(n);
    if (e != cudaSuccess) return e;
    tg.d = std::move(d); tg.h = std::move(h); tg.t = std::move(t);
    return cudaSuccess;
}

static void group_all_or_nothing() {
    Target tg;
    CHECK(fill(tg, 4) == cudaSuccess && live() == 3);
    char* d = tg.d.get(); int* h = tg.h.get(); long* t = tg.t.get();
    for (int k = 1; k <= 3; ++k) {
        g_fail_at = g_allocs + k;
        CHECK(fill(tg, 8) == cudaErrorMemoryAllocation);
        CHECK(live() == 3 && tg.d.get() == d && tg.h.get() == h && tg.t.get() == t && tg.d.cap() == 4);
    }
    CHECK(fill(tg, 8) == cudaSuccess && live() == 3 && tg.d.cap() == 8 && tg.h.cap() == 8 && tg.t.cap() == 8);
}

static void destruction_frees_live() {
    {
        Target a, empty;
        DmDev<int> arr[2];
        DmStream s;
        DmEvent unused;
        CHECK(fill(a, 4) == cudaSuccess && arr[1].alloc(3) == cudaSuccess && s.create() == cudaSuccess);
        CHECK(live() == 5 && g_frees == 0);
    }
    CHECK(live() == 0 && g_frees == 5);                   // one free per live object, none for the empty owners
    g_fail_at = g_allocs + 1;
    DmStream s;
    CHECK(s.create() == cudaErrorMemoryAllocation && s.get() == nullptr);
}

int main(int argc, char** argv) {
    const std::string c = argc > 1 ? argv[1] : "";
    if (c == "grow_within_capacity") grow_within_capacity();
    else if (c == "growth_frees_old_once") growth_frees_old_once();
    else if (c == "move_transfers") move_transfers();
    else if (c == "group_all_or_nothing") group_all_or_nothing();
    else if (c == "destruction_frees_live") destruction_frees_live();
    else { printf("unknown case %s\n", c.c_str()); return 2; }
    CHECK(live() == 0);                                   // every case's owners are gone by now
    CHECK(g_bad == 0);                                    // no free of a null or dead pointer
    printf("allocs=%d frees=%d\n", g_allocs, g_frees);
    return g_failed ? 1 : 0;
}
"""

CASES = ["grow_within_capacity", "growth_frees_old_once", "move_transfers", "group_all_or_nothing",
         "destruction_frees_live"]


def _cuda_include():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    for home in (os.environ.get("CUDA_HOME"), os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "/usr/local/cuda"):
        if home and os.path.exists(os.path.join(home, "include", "cuda_runtime.h")):
            return os.path.join(home, "include")
    return None


@pytest.fixture(scope="module")
def program(tmp_path_factory):
    inc = _cuda_include()
    if inc is None or shutil.which("g++") is None:
        pytest.skip("needs g++ and the CUDA toolkit's headers")
    d = tmp_path_factory.mktemp("dm_buf")
    src, exe = d / "dm_buf_test.cpp", d / "dm_buf_test"
    src.write_text(PROGRAM)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, "-I", inc, "-o", str(exe), str(src)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.mark.parametrize("case", CASES)
def test_dm_buf(program, case):
    r = subprocess.run([program, case], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
