// Host-side plumbing of the reference-facing entry points: a small pool of copy threads that moves a caller's
// PAGEABLE buffer (the reference hands over an ordinary Vec<f32>, decode.rs:43-49) through a ring of pinned staging
// buffers so that the H2D DMA of chunk c overlaps the memcpy of chunk c+1 -- cudaMemcpy from pageable memory is far
// below the PCIe limit (tools/hostcopy_bench.cu measures both).
// Also: CPU affinity of our own threads to the NUMA node the GPU hangs off.
#pragma once

#include <atomic>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

namespace aptb200 {

// CPUs local to the PCI device of CUDA device `device` (from /sys/bus/pci/devices/<id>/local_cpulist); empty if unknown.
std::vector<int> device_local_cpus(int device);
// Binds the calling thread to those CPUs (no-op if unknown or APTB200_NO_AFFINITY is set).  Returns true if bound.
bool bind_thread_to_device(int device);

// Persistent worker threads splitting one memcpy; one job at a time (run() blocks until the copy is done).
class CopyPool {
public:
    CopyPool(int threads, int device);
    ~CopyPool();
    CopyPool(const CopyPool &) = delete;
    CopyPool &operator=(const CopyPool &) = delete;
    void copy(void *dst, const void *src, size_t bytes);
    int threads() const { return static_cast<int>(workers_.size()) + 1; }

private:
    void worker(int index);
    std::vector<std::thread> workers_;
    std::mutex m_;
    std::condition_variable cv_start_;
    std::atomic<uint64_t> gen_atomic_{0};
    std::atomic<int> pending_{0};
    std::atomic<bool> quit_{false};
    char *dst_ = nullptr;
    const char *src_ = nullptr;
    size_t bytes_ = 0, slice_ = 0;
    int device_;
};

// Ring of pinned staging buffers + the pool: host -> device and device -> host copies of pageable buffers.
class HostStager {
public:
    HostStager(int device, size_t chunk_bytes, int ring, int threads);
    ~HostStager();
    bool ok() const { return ok_; }
    // Enqueues the upload of `bytes` from pageable `src` to device `dst` on `stream`; returns when the last chunk has
    // been handed to the DMA engine (the caller's buffer is no longer needed after return).
    cudaError_t upload(void *dst, const void *src, size_t bytes, cudaStream_t stream);
    // Enqueues the upload of `count` pieces of `piece` bytes, piece i read from pageable src + offsets[i], packed one after
    // the other at device `dst`; several pieces share a ring buffer and its one DMA.  Returns as upload() does.
    cudaError_t upload_pieces(void *dst, const void *src, const uint64_t *offsets, size_t count, size_t piece,
                              cudaStream_t stream);
    // Copies `bytes` from pinned `src` (already filled, e.g. by a finished D2H) into pageable `dst` with the pool.
    void scatter(void *dst, const void *src, size_t bytes) { pool_.copy(dst, src, bytes); }
    size_t chunk_bytes() const { return chunk_; }

private:
    int device_;
    size_t chunk_;
    std::vector<char *> ring_;
    std::vector<cudaEvent_t> ev_;
    std::vector<bool> used_;
    CopyPool pool_;
    bool ok_ = false;
};

// The staging ring of every pageable-buffer upload: three 16-MiB buffers and APTB200_COPY_THREADS copy threads (8 by
// default).  nullptr under APTB200_NO_STAGER or when the ring cannot be allocated: the caller then uses cudaMemcpyAsync.
std::unique_ptr<HostStager> make_stager(int device);

// true if `p` is ordinary pageable host memory (not pinned / registered / managed / device)
bool is_pageable(const void *p);

}  // namespace aptb200
