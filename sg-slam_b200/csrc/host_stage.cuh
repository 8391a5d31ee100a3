// host_stage.cuh -- device scratch of the host-pointer entry points (one frame, host arrays in and out).
// Kept out of sgs_common.h: that header is also compiled without CUDA into the host-check library.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "sgs_common.h"

namespace sgs {

// Declare the call's slots first, then commit(): one cudaMalloc holds them all, every slot 256-byte aligned and at least one
// byte long (so a zero-length slot still gets a distinct, valid pointer); commit() then uploads the inputs and clears the zeroed
// outputs.  Each declaration stores the slot's device pointer into *dst at commit().  The first CUDA failure is kept and reported
// once, as SGS_ERR_CUDA with set_error naming the entry point; later copies are skipped.  The allocation is freed by scope.
class HostStage {
public:
    explicit HostStage(const char* entry) : entry_(entry) {}
    ~HostStage() { if (base_) cudaFree(base_); }
    HostStage(const HostStage&) = delete;
    HostStage& operator=(const HostStage&) = delete;

    // n elements uploaded from host / left for the device to write / cleared to zero
    template <class T> void in(T** dst, const std::remove_const_t<T>* host, size_t n) { slots_.push_back({dst, host, n * sizeof(T), 0, kIn}); }
    template <class T> void out(T** dst, size_t n) { slots_.push_back({dst, nullptr, n * sizeof(T), 0, kOut}); }
    template <class T> void zeroed(T** dst, size_t n) { slots_.push_back({dst, nullptr, n * sizeof(T), 0, kZero}); }
    // an optional input: a NULL host pointer gives a NULL device pointer
    template <class T> void opt(T** dst, const std::remove_const_t<T>* host, size_t n) {
        if (host) in(dst, host, n);
        else *dst = nullptr;
    }

    int commit() {
        size_t total = 0;
        for (Slot& s : slots_) { s.off = total; total += (std::max<size_t>(s.bytes, 1) + 255) & ~size_t(255); }
        if (check(cudaMalloc(&base_, total))) return SGS_ERR_CUDA;
        for (const Slot& s : slots_) {
            void* p = static_cast<char*>(base_) + s.off;
            std::memcpy(s.dst, &p, sizeof p);
            if (err_ == cudaSuccess && s.kind == kIn && s.bytes) check(cudaMemcpy(p, s.host, s.bytes, cudaMemcpyHostToDevice));
            if (err_ == cudaSuccess && s.kind == kZero) check(cudaMemset(p, 0, s.bytes));
        }
        return status();
    }

    // synchronous copy of n elements of a device slot into caller memory
    template <class T> int to_host(T* host, const T* dev, size_t n) {
        return err_ == cudaSuccess && n ? check(cudaMemcpy(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost)) : status();
    }

    int check(cudaError_t e) {
        if (e != cudaSuccess && err_ == cudaSuccess) { err_ = e; set_error("%s: %s", entry_, cudaGetErrorString(e)); }
        return status();
    }
    int status() const { return err_ == cudaSuccess ? SGS_OK : SGS_ERR_CUDA; }

private:
    enum Kind { kIn, kOut, kZero };
    struct Slot { void* dst; const void* host; size_t bytes, off; Kind kind; };

    const char* entry_;
    std::vector<Slot> slots_;
    void* base_ = nullptr;
    cudaError_t err_ = cudaSuccess;
};

}  // namespace sgs
