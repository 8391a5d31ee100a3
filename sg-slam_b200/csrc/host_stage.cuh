// host_stage.cuh -- CUDA resources of the host side: the device scratch of the host-pointer entry points (one frame, host arrays in and
// out), the resources every long-lived handle owns, and the handles' stage timers.
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

// SGS_CUDA_TRY with the message "<entry>: <CUDA error>"
#define SGS_CUDA_TRY_AT(entry, expr)                                                                \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) { ::sgs::set_error("%s: %s", entry, cudaGetErrorString(_e)); return SGS_ERR_CUDA; } \
    } while (0)

// Everything a long-lived handle acquires from the CUDA runtime: one cudaMalloc / cudaMallocHost per buffer, non-blocking streams, events.  The
// destructor releases them in reverse order of acquisition on the handle's device; an owner that holds nothing makes no CUDA call.  A failed
// acquisition leaves its pointer NULL and records nothing.
class HandleResources {
public:
    explicit HandleResources(int device) : device_(device) {}
    ~HandleResources() {
        if (held_.empty()) return;
        cudaSetDevice(device_);
        for (auto r = held_.rbegin(); r != held_.rend(); ++r) r->release(r->p);
    }
    HandleResources(const HandleResources&) = delete;
    HandleResources& operator=(const HandleResources&) = delete;

    template <class T> cudaError_t alloc(T** p, size_t bytes) { return keep(cudaMalloc((void**)p, bytes), p, cudaFree); }
    template <class T> cudaError_t host_alloc(T** p, size_t bytes) { return keep(cudaMallocHost((void**)p, bytes), p, cudaFreeHost); }
    cudaError_t stream(cudaStream_t* s) {
        return keep(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking), s, [](void* q) { return cudaStreamDestroy((cudaStream_t)q); });
    }
    cudaError_t event(cudaEvent_t* e, unsigned flags) { return keep(cudaEventCreateWithFlags(e, flags), e, [](void* q) { return cudaEventDestroy((cudaEvent_t)q); }); }
    // a lazily grown device buffer: frees *p, then allocates `bytes`; on failure *p is NULL
    template <class T> cudaError_t regrow(T** p, size_t bytes) {
        for (auto r = held_.begin(); *p && r != held_.end(); ++r)
            if (r->p == *p) { r->release(r->p); held_.erase(r); break; }
        return alloc(p, bytes);
    }
    // a buffer grown on demand: regrows *p when *cap < bytes; *cap is 0 after a failed grow, so the next call tries again
    template <class T> cudaError_t grow(T** p, size_t* cap, size_t bytes) {
        if (*cap >= bytes) return cudaSuccess;
        *cap = 0;
        const cudaError_t e = regrow(p, bytes);
        if (e == cudaSuccess) *cap = bytes;
        return e;
    }

private:
    struct Held { void* p; cudaError_t (*release)(void*); };
    template <class P> cudaError_t keep(cudaError_t e, P* p, cudaError_t (*release)(void*)) {
        if (e != cudaSuccess) *p = nullptr;
        else if (*p) held_.push_back({(void*)*p, release});
        return e;
    }

    int device_;
    std::vector<Held> held_;
};

// Per-stage CUDA-event timing of a handle's launch path.  A timed call marks the start of each of its n stages and its end on its stream; its
// times are added to the totals at the next timed call or when the totals are read.  While timing is off, a mark costs one branch.
class StageTimer {
public:
    explicit StageTimer(int nstages = 0) : ms_(nstages, 0.0) {}

    // creates the n + 1 events (owned by `res`) on the first enable; resets the totals and the call count either way
    cudaError_t enable(HandleResources& res, bool on) {
        if (on && ev_.empty()) {
            std::vector<cudaEvent_t> ev(ms_.size() + 1);
            for (cudaEvent_t& e : ev)
                if (cudaError_t err = res.event(&e, cudaEventDefault)) return err;
            ev_.swap(ev);
        }
        on_ = on; pending_ = false; calls_ = 0;
        std::fill(ms_.begin(), ms_.end(), 0.0);
        return cudaSuccess;
    }
    bool on() const { return on_; }

    // start of a launch: folds the previous timed call; the call is timed when timing is on and `allowed`
    void begin(bool allowed = true) { timed_ = on_ && allowed; if (timed_) fold(); }
    void mark(int stage, cudaStream_t st) { if (timed_) cudaEventRecord(ev_[stage], st); }
    void end(cudaStream_t st) { if (timed_) { cudaEventRecord(ev_.back(), st); pending_ = true; } }

    // adds the pending call's stage times to the totals; on a failed wait the call stays pending
    cudaError_t fold() {
        if (!pending_) return cudaSuccess;
        cudaError_t e = cudaEventSynchronize(ev_.back());
        if (e != cudaSuccess) return e;
        for (size_t i = 0; i < ms_.size(); ++i) {
            float ms = 0;
            const cudaError_t ei = cudaEventElapsedTime(&ms, ev_[i], ev_[i + 1]);
            if (ei == cudaSuccess) ms_[i] += ms;
            else if (e == cudaSuccess) e = ei;
        }
        ++calls_;
        pending_ = false;
        return e;
    }
    const std::vector<double>& totals() const { return ms_; }
    int calls() const { return calls_; }

private:
    std::vector<cudaEvent_t> ev_;
    std::vector<double> ms_;
    int calls_ = 0;
    bool on_ = false, timed_ = false, pending_ = false;
};

}  // namespace sgs
