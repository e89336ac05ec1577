"""CPU: DevBuf (csrc/devbuf.cuh), the owner of every device buffer of the engine handles, compiled with g++ against a stub
cuda_runtime.h that counts allocations and can fail the k-th cudaMalloc: alloc, grow-only ensure, reset, move,
destruction, and a failed allocation that leaves the buffer empty and the byte count unchanged."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT

STUB = r"""
#pragma once
#include <cstddef>
#include <cstdlib>
typedef enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 } cudaError_t;
inline int g_mallocs = 0, g_frees = 0, g_live = 0, g_fail_at = -1;   // g_fail_at: 0-based index of the cudaMalloc to fail
inline cudaError_t cudaMalloc(void** p, size_t bytes) {
    if (g_mallocs++ == g_fail_at) { *p = (void*)0x1; return cudaErrorMemoryAllocation; }   // a garbage pointer, as a driver may leave
    *p = std::malloc(bytes ? bytes : 1);
    ++g_live;
    return cudaSuccess;
}
inline cudaError_t cudaFree(void* p) { ++g_frees; --g_live; std::free(p); return cudaSuccess; }
"""

MAIN = r"""
#include <cstdio>
#include <utility>
#include "devbuf.cuh"
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); return 1; } } while (0)
static long long bytes() { return (long long)engine::g_device_bytes.load(); }
int main() {
    {
        DevBuf<double> a;
        CHECK(a.data() == nullptr && a.size() == 0 && a.bytes() == 0 && bytes() == 0);
        CHECK(a.alloc(10) == cudaSuccess);
        CHECK(a.data() != nullptr && a.size() == 10 && a.bytes() == 80 && bytes() == 80 && g_live == 1);
        double* p = a;                                   // converts to the pointer it holds
        CHECK(p == a.data());
        // ensure is grow-only: same pointer when no growth
        CHECK(a.ensure(4) == cudaSuccess && a.data() == p && a.size() == 10 && g_mallocs == 1);
        CHECK(a.ensure(10) == cudaSuccess && a.data() == p && g_mallocs == 1);
        CHECK(a.ensure(11) == cudaSuccess && a.size() == 11 && bytes() == 88 && g_mallocs == 2 && g_live == 1);
        // alloc frees before it allocates, even to a smaller size
        const int frees = g_frees;
        CHECK(a.alloc(3) == cudaSuccess && a.size() == 3 && bytes() == 24 && g_frees == frees + 1 && g_live == 1);
        // move construction and assignment hand the allocation over
        DevBuf<double> b(std::move(a));
        CHECK(a.data() == nullptr && a.size() == 0 && b.size() == 3 && bytes() == 24 && g_live == 1);
        DevBuf<double> c;
        CHECK(c.alloc(5) == cudaSuccess && bytes() == 64 && g_live == 2);
        c = std::move(b);                                // c's own allocation is freed
        CHECK(b.data() == nullptr && c.size() == 3 && bytes() == 24 && g_live == 1);
        c.reset();
        CHECK(c.data() == nullptr && c.size() == 0 && bytes() == 0 && g_live == 0);
        c.reset();                                       // idempotent
        CHECK(g_live == 0 && bytes() == 0);
        DevBuf<int> d;
        CHECK(d.ensure(0) == cudaSuccess && d.data() == nullptr && g_mallocs == 4);
    }
    CHECK(g_live == 0 && bytes() == 0);
    {
        DevBuf<long long> e;                             // destruction frees
        CHECK(e.alloc(7) == cudaSuccess && bytes() == 56 && g_live == 1);
    }
    CHECK(g_live == 0 && bytes() == 0);
    {
        // a failed allocation leaves the buffer empty and the byte count unchanged
        DevBuf<double> keep, f;
        CHECK(keep.alloc(2) == cudaSuccess && bytes() == 16);
        CHECK(f.alloc(4) == cudaSuccess && bytes() == 48);
        g_fail_at = g_mallocs;
        CHECK(f.alloc(8) == cudaErrorMemoryAllocation);
        CHECK(f.data() == nullptr && f.size() == 0 && bytes() == 16 && g_live == 1);
        g_fail_at = g_mallocs;
        CHECK(f.ensure(1) == cudaErrorMemoryAllocation && f.data() == nullptr && f.size() == 0 && bytes() == 16);
        CHECK(f.ensure(1) == cudaSuccess && f.size() == 1 && bytes() == 24);   // the next attempt starts clean
        // a struct of buffers: assigning {} frees the whole group
        struct Group { DevBuf<double> u, v; bool ready = false; } g;
        CHECK(g.u.alloc(1) == cudaSuccess && g.v.alloc(1) == cudaSuccess && bytes() == 40);
        g.ready = true;
        g = {};
        CHECK(g.u.data() == nullptr && g.v.data() == nullptr && !g.ready && bytes() == 24 && g_live == 2);
    }
    CHECK(g_live == 0 && bytes() == 0);
    std::printf("OK\n");
    return 0;
}
"""


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_devbuf_with_stub_runtime(tmp_path):
    (tmp_path / "cuda_runtime.h").write_text(STUB)
    (tmp_path / "main.cpp").write_text(MAIN)
    csrc = os.path.join(ROOT, "gaussianprocesses.jl_b200", "csrc")
    exe = str(tmp_path / "devbuf_test")
    # the stub directory comes first, so devbuf.cuh's #include <cuda_runtime.h> resolves to it
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I", str(tmp_path), "-I", csrc,
                           str(tmp_path / "main.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "OK", out.stdout + out.stderr
