// wgmma_width_probe -- does one m64nNk8 tf32 wgmma over a whole output-channel tile give the same accumulator bits as N / 32 m64n32k8 wgmma over
// its 32-channel chunks?  conv1x1_tc_kernel relies on it: wide tiles issue each split term of a k-step (lo*hi, hi*lo, hi*hi) as one full-width
// wgmma, where they used to issue it chunk by chunk.  Every output element sees the same products in the same order both ways; this checks that the
// tensor core also rounds them the same way at every N.
//
// One warpgroup per trial accumulates a 64 x N tile over K = 64 (two 32-float k-blocks, eight k-steps) both ways, from operands laid out as in the
// kernel (activation fragments split to TF32 hi + lo in registers, weight hi / lo tiles K-major with the 128-byte swizzle in shared memory), on
// random FP32 data with subnormals, signed zeros and exponents from 2^-60 to 2^60.  Prints one line per N and exits with 0 when every N matches
// bit for bit and both ways stay within FP32-grade accuracy of a float64 sum (so that a probe computing nothing cannot pass).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "conv1x1_tc.cuh"

using namespace sgs::tc;

constexpr int kRows = 64, kKB = 2, kK = kKB * 32, kTrials = 4;

// FULL = false: the chunked issue, true: the full-width issue (one launch each: both accumulators at once would not fit the registers at N = 256)
template <int NC, bool FULL>
__global__ void __launch_bounds__(128) probe_kernel(const float* __restrict__ X, const float* __restrict__ Whi, const float* __restrict__ Wlo,
                                                    float* __restrict__ out) {
    constexpr int NT = NC * kWN, ROWB = 128, b_bytes = NT * ROWB;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t sbase = (smem_addr(smem_raw) + 1023u) & ~1023u;
    uint8_t* gbase = smem_raw + (sbase - smem_addr(smem_raw));
    const int trial = blockIdx.x;
    X += (size_t)trial * kRows * kK; Whi += (size_t)trial * NT * kK; Wlo += (size_t)trial * NT * kK;
    // weights: k-block kb at kb * 2 * b_bytes, hi then lo, element (n, k) where TMA's 128-byte swizzle puts it
    for (int i = threadIdx.x; i < kKB * NT * 32; i += blockDim.x) {
        const int kb = i / (NT * 32), n = (i / 32) % NT, k = i % 32;
        const uint32_t o = kb * 2 * b_bytes + swz_offset<ROWB>(n, k);
        *reinterpret_cast<float*>(gbase + o) = Whi[(size_t)n * kK + kb * 32 + k];
        *reinterpret_cast<float*>(gbase + o + b_bytes) = Wlo[(size_t)n * kK + kb * 32 + k];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> wgmma operand reads
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int r0 = 16 * warp + g;
    float acc_c[FULL ? 1 : NC][16], acc_f[FULL ? NT / 2 : 1];
#pragma unroll
    for (int c = 0; c < (FULL ? 1 : NC); ++c)
#pragma unroll
        for (int i = 0; i < 16; ++i) acc_c[c][i] = 0.f;
#pragma unroll
    for (int i = 0; i < (FULL ? NT / 2 : 1); ++i) acc_f[i] = 0.f;
    for (int kb = 0; kb < kKB; ++kb) {
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = kb * 32 + 8 * j + t;
            split_tf32(__float_as_uint(X[r0 * kK + k]), ah[j][0], al[j][0]);
            split_tf32(__float_as_uint(X[(r0 + 8) * kK + k]), ah[j][1], al[j][1]);
            split_tf32(__float_as_uint(X[r0 * kK + k + 4]), ah[j][2], al[j][2]);
            split_tf32(__float_as_uint(X[(r0 + 8) * kK + k + 4]), ah[j][3], al[j][3]);
        }
        const uint32_t bh0 = sbase + (uint32_t)kb * 2 * b_bytes;
        wgmma_fence();
        if constexpr (!FULL) {
            // the chunked issue: per k-step, the three terms on each 32-channel chunk in turn
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int c = 0; c < NC; ++c) {
                    const uint32_t b = bh0 + (uint32_t)(c * kWN * ROWB + j * 32);
                    wgmma_tf32<32>(acc_c[c], al[j], kmajor_desc<ROWB>(b));
                    wgmma_tf32<32>(acc_c[c], ah[j], kmajor_desc<ROWB>(b + b_bytes));
                    wgmma_tf32<32>(acc_c[c], ah[j], kmajor_desc<ROWB>(b));
                }
        } else {
            // the full-width issue: per k-step, each term once over all NT channels
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t b = bh0 + (uint32_t)(j * 32);
                wgmma_tf32<NT>(acc_f, al[j], kmajor_desc<ROWB>(b));
                wgmma_tf32<NT>(acc_f, ah[j], kmajor_desc<ROWB>(b + b_bytes));
                wgmma_tf32<NT>(acc_f, ah[j], kmajor_desc<ROWB>(b));
            }
        }
        wgmma_commit();
        wgmma_wait_all();
    }
    // both written to [row][channel] through their own register maps: chunk c, acc_c[c][4j + 2h + q] is channel 32c + 8j + 2t + q of row r0 + 8h;
    // acc_f[4j + 2h + q] is channel 8j + 2t + q
    out += (size_t)trial * kRows * NT;
    if constexpr (!FULL) {
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
            for (int i = 0; i < 16; ++i) out[(r0 + 8 * ((i >> 1) & 1)) * NT + 32 * c + 8 * (i >> 2) + 2 * t + (i & 1)] = acc_c[c][i];
    } else {
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) out[(r0 + 8 * ((i >> 1) & 1)) * NT + 8 * (i >> 2) + 2 * t + (i & 1)] = acc_f[i];
    }
}

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static uint64_t next_u64() {                    // splitmix64
    uint64_t z = (rng_state += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull; z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
// random operand: 4 % signed zeros, 6 % subnormals, 10 % exponents in [-60, 60], the rest in [-8, 8]; random sign and 23-bit mantissa
static float random_operand() {
    const uint64_t r = next_u64();
    const uint32_t sign = (uint32_t)(r >> 63) << 31, mant = (uint32_t)(r >> 8) & 0x7fffffu;
    const int pick = (int)(r % 100);
    uint32_t bits;
    if (pick < 4) bits = sign;
    else if (pick < 10) bits = sign | (mant ? mant : 1u);
    else {
        const int e = pick < 20 ? (int)((r >> 40) % 121) - 60 : (int)((r >> 40) % 17) - 8;
        bits = sign | ((uint32_t)(e + 127) << 23) | mant;
    }
    float f; memcpy(&f, &bits, 4);
    return f;
}

#define CHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); return false; } } while (0)

template <int NC>
static bool run_width(bool* ok) {
    constexpr int NT = NC * kWN;
    std::vector<float> X((size_t)kTrials * kRows * kK), W((size_t)kTrials * NT * kK), Wh(W.size()), Wl(W.size());
    for (float& x : X) x = random_operand();
    for (size_t i = 0; i < W.size(); ++i) { W[i] = random_operand(); split_tf32_host(W[i], Wh[i], Wl[i]); }
    const size_t nout = (size_t)kTrials * kRows * NT;
    float *dX, *dWh, *dWl, *dC, *dF;
    CHECK(cudaMalloc(&dX, X.size() * 4)); CHECK(cudaMalloc(&dWh, W.size() * 4)); CHECK(cudaMalloc(&dWl, W.size() * 4));
    CHECK(cudaMalloc(&dC, nout * 4)); CHECK(cudaMalloc(&dF, nout * 4));
    CHECK(cudaMemcpy(dX, X.data(), X.size() * 4, cudaMemcpyHostToDevice));
    CHECK(cudaMemcpy(dWh, Wh.data(), W.size() * 4, cudaMemcpyHostToDevice));
    CHECK(cudaMemcpy(dWl, Wl.data(), W.size() * 4, cudaMemcpyHostToDevice));
    CHECK(cudaMemset(dC, 0xff, nout * 4)); CHECK(cudaMemset(dF, 0xff, nout * 4));
    const int smem = kKB * 2 * NT * 128 + 1024;
    CHECK(cudaFuncSetAttribute(probe_kernel<NC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CHECK(cudaFuncSetAttribute(probe_kernel<NC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    probe_kernel<NC, false><<<kTrials, 128, smem>>>(dX, dWh, dWl, dC);
    probe_kernel<NC, true><<<kTrials, 128, smem>>>(dX, dWh, dWl, dF);
    CHECK(cudaGetLastError());
    CHECK(cudaDeviceSynchronize());
    std::vector<float> C(nout), F(nout);
    CHECK(cudaMemcpy(C.data(), dC, nout * 4, cudaMemcpyDeviceToHost));
    CHECK(cudaMemcpy(F.data(), dF, nout * 4, cudaMemcpyDeviceToHost));
    cudaFree(dX); cudaFree(dWh); cudaFree(dWl); cudaFree(dC); cudaFree(dF);
    size_t differ = 0, zeros = 0, subn = 0;
    double worst = 0;
    for (int tr = 0; tr < kTrials; ++tr)
        for (int r = 0; r < kRows; ++r)
            for (int n = 0; n < NT; ++n) {
                const size_t o = ((size_t)tr * kRows + r) * NT + n;
                if (memcmp(&C[o], &F[o], 4)) ++differ;
                if (C[o] == 0.f) ++zeros;
                if (C[o] != 0.f && std::fabs(C[o]) < 1.17549435e-38f) ++subn;
                double ref = 0, s = 0;
                for (int k = 0; k < kK; ++k) {
                    const double p = (double)X[((size_t)tr * kRows + r) * kK + k] * (double)W[((size_t)tr * NT + n) * kK + k];
                    ref += p; s += std::fabs(p);
                }
                if (s > 0) worst = std::fmax(worst, std::fmax(std::fabs(C[o] - ref), std::fabs(F[o] - ref)) / s);
                else if (C[o] != 0.f || F[o] != 0.f) worst = 1;
            }
    const bool pass = differ == 0 && worst < 1e-4;
    printf("N=%d elements=%zu differing=%zu zeros=%zu subnormal=%zu max_err_over_S=%.3g %s\n", NT, nout, differ, zeros, subn, worst, pass ? "ok" : "FAIL");
    *ok = *ok && pass;
    return true;
}

int main() {
    bool ok = true;
    if (!(run_width<1>(&ok) && run_width<2>(&ok) && run_width<3>(&ok) && run_width<4>(&ok) && run_width<5>(&ok) && run_width<6>(&ok) &&
          run_width<7>(&ok) && run_width<8>(&ok)))
        return 2;
    printf(ok ? "all widths match bit for bit\n" : "MISMATCH\n");
    return ok ? 0 : 1;
}
