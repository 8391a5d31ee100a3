// gemm_tile_trace -- where the time of one conv1x1_tc_kernel tile goes.  Built with -DSGS_GEMM_TRACE (tools/gemm_tile_trace.py does it), the
// kernel writes clock64() stamps of the first tiles of CTA (0, 0) to g_gemm_trace: per consumer warpgroup the tile start, the clocks spent in
// ring waits, the last wgmma issued, its wait_group done, the epilogue done, and the clocks spent in the k-loop's wait_group; per producer the
// clocks spent waiting for free ring slots.
//
//   gemm_tile_trace Cin Cout H W frames tail      (tail 0: none, 1: hard-swish, the expansions' tail)
//
// One GEMM of the layer's shape on seeded data, planned as the detector plans it for that batch; prints one JSON line: the plan, the mean time of
// a call (CUDA events over 20 calls) and the stamps of the traced tiles (rows: warpgroup 0, warpgroup 1, producer).
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "conv1x1_tc.cuh"

using namespace sgs::tc;

struct HswishTail {
    int on;
    template <int N>
    __device__ __forceinline__ void run(float (&v)[N], int64_t) const {
        if (!on) return;
#pragma unroll
        for (int q = 0; q < N; ++q) v[q] = div6(__fmul_rn(v[q], fminf(fmaxf(__fadd_rn(v[q], 3.f), 0.f), 6.f)));
    }
};

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

int main(int argc, char** argv) {
    if (argc != 7) { fprintf(stderr, "usage: gemm_tile_trace Cin Cout H W frames tail\n"); return 2; }
    const int Cin = atoi(argv[1]), Cout = atoi(argv[2]), H = atoi(argv[3]), W = atoi(argv[4]), F = atoi(argv[5]), tail = atoi(argv[6]);
    const int npix = F * H * W;
    sgs::HandleResources res(0);
    std::vector<float> w((size_t)Cout * Cin), x((size_t)npix * Cin), b(Cout);
    uint32_t s = 12345u;
    auto rnd = [&]() { s = s * 1664525u + 1013904223u; return (float)((s >> 8) & 0xffff) / 65536.f - 0.5f; };
    for (auto& v : w) v = rnd();
    for (auto& v : x) v = rnd();
    for (auto& v : b) v = rnd();
    GemmPlan P;
    if (!plan_weights(res, w.data(), Cin, Cout, &P, 0, (npix + kBM - 1) / kBM)) { fprintf(stderr, "plan_weights failed\n"); return 1; }
    float *dx = nullptr, *db = nullptr, *dout = nullptr;
    CK(res.alloc(&dx, x.size() * 4)); CK(res.alloc(&db, b.size() * 4)); CK(res.alloc(&dout, (size_t)npix * Cout * 4));
    CK(cudaMemcpy(dx, x.data(), x.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(db, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
    CUtensorMap mapA;
    if (!encode_kmajor_map(&mapA, dx, npix, Cin, Cin, kBM, P.BK)) { fprintf(stderr, "encode_kmajor_map failed\n"); return 1; }
    const HswishTail epi{tail};
    auto launch = [&]() { return launch_conv1x1_tc_map(P, mapA, npix, db, dout, H * W, (int64_t)H * W * Cout, 0, Cout, epi, 0); };
    for (int i = 0; i < 3; ++i) if (!launch()) { fprintf(stderr, "launch failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
    CK(cudaDeviceSynchronize());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const int calls = 20;
    CK(cudaEventRecord(e0));
    for (int i = 0; i < calls; ++i) launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    static long long zero[3][kTraceTiles][TR_EVENTS];
    CK(cudaMemcpyToSymbol(g_gemm_trace, zero, sizeof(zero)));
    launch();
    CK(cudaDeviceSynchronize());
    static long long tr[3][kTraceTiles][TR_EVENTS];
    CK(cudaMemcpyFromSymbol(tr, g_gemm_trace, sizeof(tr)));
    int gx = sm_count() * (P.NT <= kNarrowChunks * kWN ? 2 : 1) / P.n_tiles;
    const int m_tiles = (npix + kBM - 1) / kBM;
    if (gx > m_tiles) gx = m_tiles;
    printf("{\"cin\": %d, \"cout\": %d, \"h\": %d, \"w\": %d, \"frames\": %d, \"nt\": %d, \"n_tiles\": %d, \"kb\": %d, \"bk\": %d, \"stages\": %d, "
           "\"wres\": %d, \"grid_x\": %d, \"m_tiles\": %d, \"ms\": %.5f, \"trace\": [", Cin, Cout, H, W, F, P.NT, P.n_tiles, P.KB, P.BK, P.stages,
           P.b_resident, gx, m_tiles, ms / calls);
    for (int r = 0; r < 3; ++r) {
        printf(r ? ", [" : "[");
        for (int t = 0; t < kTraceTiles; ++t) {
            printf(t ? ", [" : "[");
            for (int e = 0; e < TR_EVENTS; ++e) printf(e ? ", %lld" : "%lld", tr[r][t][e]);
            printf("]");
        }
        printf("]");
    }
    printf("]}\n");
    return 0;
}
