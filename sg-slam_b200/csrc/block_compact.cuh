// block_compact.cuh -- block-wide ordered compaction: the elements a block keeps get consecutive output positions in their input order.
#pragma once
#include <cuda_runtime.h>

namespace sgs {

// Called by every thread of a block of kThreads threads, once per chunk of kThreads consecutive elements (thread t holds element t of the chunk).
// Returns the output position of the thread's element, -1 when it is not kept, and adds the chunk's kept elements to `count`: the number kept
// so far, the same in every thread (start it at 0).  What the caller stores at the positions is visible to other threads after its next
// __syncthreads().
template <int kThreads>
__device__ __forceinline__ int block_ordered_slot(bool keep, int& count) {
    static_assert(kThreads % 32 == 0, "whole warps");
    __shared__ int warp_kept[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_kept[warp] = __popc(bal);
    __syncthreads();
    int before = count;
    for (int w = 0; w < kThreads / 32; ++w) {
        if (w < warp) before += warp_kept[w];
        count += warp_kept[w];
    }
    __syncthreads();        // every warp has read warp_kept before the next chunk writes it
    return keep ? before + __popc(bal & ((1u << lane) - 1u)) : -1;
}

}  // namespace sgs
