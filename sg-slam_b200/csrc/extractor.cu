// extractor.cu -- host side of the batched ORB extractor handle (sgs_extractor_* entry points of include/sgs_abi.h).
// Owns the device buffers laid out for `max_batch` frames of one geometry and enqueues the kernel pipeline of
// extract_kernels.cu on one stream.  Replaces ORB_SLAM2::ORBextractor (include/ORBextractor.h:45-105).
#include <cuda_runtime.h>

#include <algorithm>

#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "extract_kernels.h"
#include "host_stage.cuh"

using namespace sgs;

struct sgs_extractor {
    explicit sgs_extractor(int dev) : device(dev), res(dev) {}
    OrbPlan plan;
    int device;
    HandleResources res;
    int max_batch = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;      // host -> device copies of the chunked host path run here, ahead of the kernels
    cudaEvent_t chunk_ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t chunk_done = nullptr;
    DevPlan dev{};                 // template; nframes / level-0 pointers patched per call
    // device allocations
    uint8_t* d_pyr = nullptr;      // own pyramid: levels 0..L-1, each [max_batch][h][pitch]
    uint8_t* d_blur = nullptr;
    uint32_t* d_cand = nullptr;
    int32_t* d_cand_count = nullptr;
    uint32_t* d_kp_stage = nullptr;
    int32_t* d_kp_stage_n = nullptr;
    sgs_keypoint* d_out_kps = nullptr;
    uint8_t* d_out_desc = nullptr;
    int32_t* d_out_count = nullptr;
    int32_t* d_error = nullptr;
    FastCell* d_cells = nullptr;
    short4* d_tabs = nullptr;
    uint64_t* d_key_scratch = nullptr;
    int64_t* d_key_scratch_off = nullptr;
    int64_t key_scratch_fstride = 0;
    std::vector<int64_t> lvl_off;  // byte offset of level l (frame 0) inside d_pyr / d_blur
    int smem_key_cap = 0, node_cap = 0;
    size_t qt_smem = 0;
    FastLaunchPlan fast_plan;
    FastTmaMaps fast_maps{};
    bool maps_ok = false;            // levels >= 1 (own buffers) encoded
    const void* map0_ptr = nullptr; int map0_pitch = 0; int64_t map0_fstride = 0; int map0_frames = 0; bool map0_ok = false;
    // pinned staging for the host API
    uint8_t* h_in = nullptr; size_t h_in_bytes = 0;
    sgs_keypoint* h_kps = nullptr; uint8_t* h_desc = nullptr; int32_t* h_count = nullptr; int32_t* h_error = nullptr;
    int last_nframes = 0;
    bool last_level0_external = false;
    // optional per-stage timing (CUDA events on the launching stream): pyramid, FAST, quadtree, blur, describe
    StageTimer timer{5};
    cudaStream_t last_stream = nullptr;
};

namespace {

int fail_invalid(const char* msg) { set_error("%s", msg); return SGS_ERR_INVALID; }

// Enqueue the whole pipeline for frames [frame0, frame0 + nframes) of a batch whose level 0 is (d_l0, pitch, fstride).  A chunk
// (frame0 > 0 or fewer frames than the batch) works on the same buffers through shifted base pointers; only the TMA tensor maps
// keep addressing the whole batch (`map_frames` frames) and take frame0 as a coordinate offset.
int enqueue(sgs_extractor* ex, const uint8_t* d_l0, int pitch, int64_t fstride, int nframes, cudaStream_t st, int frame0 = 0, int map_frames = 0,
            bool allow_prof = true) {
    DevPlan P = ex->dev;
    P.nframes = nframes;
    P.lv[0].img = d_l0; P.lv[0].pitch = pitch; P.lv[0].fstride = fstride;
    const int L = P.nlevels;
    if (map_frames <= 0) map_frames = frame0 + nframes;
    uint64_t* key_scratch = ex->d_key_scratch;
    if (frame0 > 0) {
        for (int l = 0; l < L; ++l) {
            DevLevel& v = P.lv[l];
            v.img += (int64_t)frame0 * v.fstride;
            if (v.img_w) v.img_w += (int64_t)frame0 * v.fstride;
            v.blur += (int64_t)frame0 * v.bfstride;
            v.cand += (int64_t)frame0 * P.cand_fstride;
        }
        P.cand_count += (int64_t)frame0 * L; P.kp_stage += (int64_t)frame0 * P.kp_stage_per_frame; P.kp_stage_n += (int64_t)frame0 * L;
        P.out_kps += (int64_t)frame0 * P.out_cap; P.out_desc += (int64_t)frame0 * P.out_cap * 32; P.out_count += frame0;
        if (key_scratch) key_scratch += (int64_t)frame0 * ex->key_scratch_fstride;
    }
    StageTimer& T = ex->timer;
    T.begin(allow_prof);
    SGS_CUDA_TRY(cudaMemsetAsync(P.cand_count, 0, sizeof(int32_t) * (size_t)nframes * L, st));
    T.mark(0, st);
    for (int l = 1; l < L; ++l) {
        if (resize_tile_supported(P, l)) launch_resize_tile(P, l, st); else launch_resize(P, l, st);
    }
    T.mark(1, st);
    {   // tiles by TMA when every level could be described by a tensor map (16-byte aligned base / pitch); the same kernel with plain loads otherwise
        bool tma = ex->maps_ok;
        if (tma && !(ex->map0_ok && ex->map0_ptr == d_l0 && ex->map0_pitch == pitch && ex->map0_fstride == fstride && ex->map0_frames >= map_frames)) {
            ex->map0_ok = encode_level_map(&ex->fast_maps.m[0], d_l0, P.lv[0].w, P.lv[0].h, pitch, fstride, map_frames, ex->fast_plan.tp, ex->fast_plan.th);
            ex->map0_ptr = d_l0; ex->map0_pitch = pitch; ex->map0_fstride = fstride; ex->map0_frames = map_frames;
        }
        launch_fast_v2(P, ex->fast_maps, tma && ex->map0_ok, ex->fast_plan, ex->d_cells, (int)ex->plan.cells.size(), frame0, st);
    }
    T.mark(2, st);
    launch_quadtree(P, ex->smem_key_cap, ex->node_cap, ex->qt_smem, key_scratch, ex->key_scratch_fstride, ex->d_key_scratch_off, st);
    T.mark(3, st);
    launch_blur_all(P, st);
    T.mark(4, st);
    launch_describe(P, st);
    T.end(st);
    SGS_CUDA_TRY(cudaGetLastError());
    ex->last_nframes = frame0 + nframes;
    ex->last_stream = st;
    return SGS_OK;
}

}  // namespace

extern "C" {

SGS_API int sgs_abi_version(void) { return SGS_ABI_VERSION; }
SGS_API const char* sgs_last_error(void) { return sgs::last_error_cstr(); }

SGS_API int sgs_device_count(int* n) {
    if (!n) return fail_invalid("sgs_device_count: NULL");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) { *n = 0; set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e)); return SGS_ERR_CUDA; }
    *n = c;
    return SGS_OK;
}

SGS_API int sgs_extractor_create(const sgs_orb_params* params, int width, int height, int max_batch, int device, sgs_extractor** out) {
    if (!params || !out) return fail_invalid("sgs_extractor_create: NULL argument");
    if (max_batch < 1 || max_batch > 65535) return fail_invalid("sgs_extractor_create: max_batch outside [1,65535]");
    *out = nullptr;
    auto ex = std::make_unique<sgs_extractor>(device);
    int st = make_plan(*params, width, height, &ex->plan);
    if (st != SGS_OK) return st;
    ex->max_batch = max_batch;
    HandleResources& R = ex->res;
    SGS_CUDA_TRY(cudaSetDevice(device));
    SGS_CUDA_TRY(R.stream(&ex->stream));
    SGS_CUDA_TRY(R.stream(&ex->copy_stream));
    for (auto& e : ex->chunk_ev) SGS_CUDA_TRY(R.event(&e, cudaEventDisableTiming));
    SGS_CUDA_TRY(R.event(&ex->chunk_done, cudaEventDisableTiming));
    const OrbPlan& PL = ex->plan;
    const int L = PL.nlevels;
    const int64_t B = max_batch;
    // pyramid + blurred pyramid: level-major, frames contiguous inside a level
    ex->lvl_off.assign(L, 0);
    int64_t total = 0;
    for (int l = 0; l < L; ++l) { ex->lvl_off[l] = total; total += B * PL.lv[l].frame_stride; }
    SGS_CUDA_TRY(R.alloc(&ex->d_pyr, (size_t)total + 256));
    SGS_CUDA_TRY(R.alloc(&ex->d_blur, (size_t)total + 256));
    SGS_CUDA_TRY(R.alloc(&ex->d_cand, sizeof(uint32_t) * (size_t)(B * PL.cand_per_frame)));
    SGS_CUDA_TRY(R.alloc(&ex->d_cand_count, sizeof(int32_t) * (size_t)(B * L)));
    SGS_CUDA_TRY(R.alloc(&ex->d_kp_stage, sizeof(uint32_t) * (size_t)(B * PL.max_kp_per_frame)));
    SGS_CUDA_TRY(R.alloc(&ex->d_kp_stage_n, sizeof(int32_t) * (size_t)(B * L)));
    SGS_CUDA_TRY(R.alloc(&ex->d_out_kps, sizeof(sgs_keypoint) * (size_t)(B * PL.max_kp_per_frame)));
    SGS_CUDA_TRY(R.alloc(&ex->d_out_desc, (size_t)(B * PL.max_kp_per_frame) * 32));
    SGS_CUDA_TRY(R.alloc(&ex->d_out_count, sizeof(int32_t) * (size_t)B));
    SGS_CUDA_TRY(R.alloc(&ex->d_error, sizeof(int32_t)));
    SGS_CUDA_TRY(cudaMemset(ex->d_error, 0, sizeof(int32_t)));
    SGS_CUDA_TRY(cudaMemset(ex->d_out_count, 0, sizeof(int32_t) * (size_t)B));
    SGS_CUDA_TRY(R.alloc(&ex->d_cells, sizeof(FastCell) * PL.cells.size()));
    SGS_CUDA_TRY(cudaMemcpy(ex->d_cells, PL.cells.data(), sizeof(FastCell) * PL.cells.size(), cudaMemcpyHostToDevice));
    // bilinear tables
    size_t ntab = 0;
    for (int l = 1; l < L; ++l) ntab += PL.xtab[l].size() / 4 + PL.ytab[l].size() / 4;
    SGS_CUDA_TRY(R.alloc(&ex->d_tabs, sizeof(short4) * (ntab + 1)));
    {
        std::vector<short4> h(ntab + 1);
        size_t o = 0;
        for (int l = 1; l < L; ++l) {
            for (int pass = 0; pass < 2; ++pass) {
                const std::vector<int16_t>& t = pass ? PL.ytab[l] : PL.xtab[l];
                for (size_t i = 0; i < t.size() / 4; ++i) h[o + i] = make_short4(t[4 * i], t[4 * i + 1], t[4 * i + 2], 0);
                if (pass) ex->dev.lv[l].ytab = ex->d_tabs + o; else ex->dev.lv[l].xtab = ex->d_tabs + o;
                o += t.size() / 4;
            }
        }
        SGS_CUDA_TRY(cudaMemcpy(ex->d_tabs, h.data(), sizeof(short4) * ntab, cudaMemcpyHostToDevice));
    }
    // quadtree: shared-memory budget and the global fallback for the sort keys
    ex->node_cap = 0;
    for (int l = 0; l < L; ++l) {
        const int c = qt_pool_cap(PL.lv[l].n_target, PL.lv[l].n_ini);
        if (c > ex->node_cap) ex->node_cap = c;
    }
    const size_t node_bytes = (quadtree_node_bytes(ex->node_cap) + 15) & ~(size_t)15;
    const size_t smem_limit = 200 * 1024;
    if (node_bytes + 1024 * 8 > smem_limit) { set_error("nfeatures too large for the shared-memory quadtree (node arrays need %zu bytes)", node_bytes); return SGS_ERR_UNSUPPORTED; }
    ex->smem_key_cap = 4096;
    while (node_bytes + (size_t)ex->smem_key_cap * 8 > 96 * 1024 && ex->smem_key_cap > 1024) ex->smem_key_cap >>= 1;
    ex->qt_smem = node_bytes + (size_t)ex->smem_key_cap * 8;
    SGS_CUDA_TRY(configure_quadtree_smem(ex->qt_smem));
    {
        std::vector<int64_t> off(L);
        int64_t o = 0;
        for (int l = 0; l < L; ++l) {
            int64_t ns = 1; while (ns < PL.lv[l].cand_cap) ns <<= 1;
            off[l] = o; o += ns;
        }
        ex->key_scratch_fstride = o;
        SGS_CUDA_TRY(R.alloc(&ex->d_key_scratch, sizeof(uint64_t) * (size_t)(B * o)));
        SGS_CUDA_TRY(R.alloc(&ex->d_key_scratch_off, sizeof(int64_t) * L));
        SGS_CUDA_TRY(cudaMemcpy(ex->d_key_scratch_off, off.data(), sizeof(int64_t) * L, cudaMemcpyHostToDevice));
    }
    // device plan template
    DevPlan& D = ex->dev;
    D.nlevels = L; D.nframes = 0; D.ini_th = params->ini_th_fast; D.min_th = params->min_th_fast;
    D.cand_fstride = PL.cand_per_frame; D.kp_stage_per_frame = PL.max_kp_per_frame; D.out_cap = PL.max_kp_per_frame;
    D.cand_count = ex->d_cand_count; D.kp_stage = ex->d_kp_stage; D.kp_stage_n = ex->d_kp_stage_n;
    D.out_kps = ex->d_out_kps; D.out_desc = ex->d_out_desc; D.out_count = ex->d_out_count; D.error_flag = ex->d_error;
    for (int i = 0; i <= kHalfPatch; ++i) D.umax[i] = PL.umax[i];
    int kp_off = 0;
    for (int l = 0; l < L; ++l) {
        const LevelGeom& g = PL.lv[l];
        DevLevel& d = D.lv[l];
        d.img = ex->d_pyr + ex->lvl_off[l]; d.img_w = ex->d_pyr + ex->lvl_off[l]; d.blur = ex->d_blur + ex->lvl_off[l];
        d.w = g.w; d.h = g.h; d.pitch = g.pitch; d.bpitch = g.pitch; d.fstride = g.frame_stride; d.bfstride = g.frame_stride;
        d.cand = ex->d_cand + g.cand_off; d.cand_cap = g.cand_cap; d.kp_cap = g.kp_cap; d.kp_off = kp_off; kp_off += g.kp_cap;
        d.max_bx = g.max_bx; d.max_by = g.max_by;
        d.qt.n_ini = g.n_ini; d.qt.h_x = g.h_x; d.qt.root_h = g.max_by - kMinBorder; d.qt.n_cols = g.n_cols; d.qt.w_cell = g.w_cell;
        d.qt.h_cell = g.h_cell; d.qt.n_target = g.n_target;
        d.scale = g.scale; d.patch_size = g.patch_size;
    }
    // warp-per-cell FAST: tile geometry, shared-memory opt-in, TMA tensor maps of the own pyramid levels
    ex->fast_plan = make_fast_launch_plan(PL);
    if (ex->fast_plan.smem_bytes > 200 * 1024) { set_error("sgs_extractor_create: FAST cells of this geometry need %d bytes of shared memory per block", ex->fast_plan.smem_bytes); return SGS_ERR_UNSUPPORTED; }
    SGS_CUDA_TRY(configure_fast_smem(ex->fast_plan.smem_bytes));
    ex->maps_ok = true;
    for (int l = 1; l < L && ex->maps_ok; ++l)
        ex->maps_ok = encode_level_map(&ex->fast_maps.m[l], D.lv[l].img, D.lv[l].w, D.lv[l].h, D.lv[l].pitch, D.lv[l].fstride, max_batch, ex->fast_plan.tp, ex->fast_plan.th);
    // pinned result staging
    SGS_CUDA_TRY(R.host_alloc(&ex->h_kps, sizeof(sgs_keypoint) * (size_t)(B * PL.max_kp_per_frame)));
    SGS_CUDA_TRY(R.host_alloc(&ex->h_desc, (size_t)(B * PL.max_kp_per_frame) * 32));
    SGS_CUDA_TRY(R.host_alloc(&ex->h_count, sizeof(int32_t) * (size_t)B));
    SGS_CUDA_TRY(R.host_alloc(&ex->h_error, sizeof(int32_t)));
    ex->h_in_bytes = (size_t)(B * PL.lv[0].frame_stride);
    SGS_CUDA_TRY(R.host_alloc(&ex->h_in, ex->h_in_bytes));
    *out = ex.release();
    return SGS_OK;
}

SGS_API void sgs_extractor_destroy(sgs_extractor* ex) { delete ex; }

SGS_API int sgs_extractor_set_profiling(sgs_extractor* ex, int enable) {
    if (!ex) return fail_invalid("sgs_extractor_set_profiling: NULL handle");
    SGS_CUDA_TRY(cudaSetDevice(ex->device));
    SGS_CUDA_TRY(ex->timer.enable(ex->res, enable != 0));
    return SGS_OK;
}

SGS_API int sgs_extractor_stage_times(sgs_extractor* ex, double* ms_total5, int* ncalls) {
    if (!ex || !ms_total5 || !ncalls) return fail_invalid("sgs_extractor_stage_times: NULL");
    SGS_CUDA_TRY(ex->timer.fold());
    for (int i = 0; i < 5; ++i) ms_total5[i] = ex->timer.totals()[i];
    *ncalls = ex->timer.calls();
    return SGS_OK;
}

SGS_API int sgs_extractor_tables(const sgs_extractor* ex, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2, int32_t* fpl) {
    if (!ex) return fail_invalid("sgs_extractor_tables: NULL handle");
    for (int l = 0; l < ex->plan.nlevels; ++l) {
        if (scale) scale[l] = ex->plan.scale[l];
        if (inv_scale) inv_scale[l] = ex->plan.inv_scale[l];
        if (sigma2) sigma2[l] = ex->plan.sigma2[l];
        if (inv_sigma2) inv_sigma2[l] = ex->plan.inv_sigma2[l];
        if (fpl) fpl[l] = ex->plan.n_per_level[l];
    }
    return SGS_OK;
}

SGS_API int sgs_extractor_max_keypoints(const sgs_extractor* ex, int* cap) {
    if (!ex || !cap) return fail_invalid("sgs_extractor_max_keypoints: NULL");
    *cap = ex->plan.max_kp_per_frame;
    return SGS_OK;
}

SGS_API int sgs_extractor_level_info(const sgs_extractor* ex, int level, int* width, int* height, int* pitch) {
    if (!ex || level < 0 || level >= ex->plan.nlevels) return fail_invalid("sgs_extractor_level_info: bad level");
    if (width) *width = ex->plan.lv[level].w;
    if (height) *height = ex->plan.lv[level].h;
    if (pitch) *pitch = ex->plan.lv[level].pitch;
    return SGS_OK;
}

SGS_API int sgs_extract_batch_device(sgs_extractor* ex, const uint8_t* d_gray, int nframes, size_t frame_stride, int pitch, void* stream) {
    if (!ex || !d_gray) return fail_invalid("sgs_extract_batch_device: NULL argument");
    if (nframes < 1 || nframes > ex->max_batch) return fail_invalid("sgs_extract_batch_device: nframes outside [1,max_batch]");
    if (pitch < ex->plan.width || frame_stride < (size_t)pitch * ex->plan.height) return fail_invalid("sgs_extract_batch_device: pitch/frame_stride too small");
    SGS_CUDA_TRY(cudaSetDevice(ex->device));
    ex->last_level0_external = true;
    return enqueue(ex, d_gray, pitch, (int64_t)frame_stride, nframes, stream ? (cudaStream_t)stream : ex->stream);
}

SGS_API int sgs_extractor_results_device(const sgs_extractor* ex, const sgs_keypoint** d_kps, const uint8_t** d_desc, const int32_t** d_counts, int* cap) {
    if (!ex) return fail_invalid("sgs_extractor_results_device: NULL handle");
    if (d_kps) *d_kps = ex->d_out_kps;
    if (d_desc) *d_desc = ex->d_out_desc;
    if (d_counts) *d_counts = ex->d_out_count;
    if (cap) *cap = ex->plan.max_kp_per_frame;
    return SGS_OK;
}

SGS_API int sgs_extractor_fetch(sgs_extractor* ex, int nframes, sgs_keypoint* kps, uint8_t* desc, int cap, int* n, void* stream) {
    if (!ex || !kps || !n) return fail_invalid("sgs_extractor_fetch: NULL argument");     // desc may be NULL: keypoints only
    if (nframes < 1 || nframes > ex->last_nframes) return fail_invalid("sgs_extractor_fetch: nframes exceeds the last call");
    SGS_CUDA_TRY(cudaSetDevice(ex->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ex->stream;
    const size_t K = (size_t)ex->plan.max_kp_per_frame;
    // pinned caller buffers with the handle's own row capacity receive the device arrays directly (no staging copy)
    cudaPointerAttributes ak, ad;
    bool direct = (size_t)cap == K && cudaPointerGetAttributes(&ak, kps) == cudaSuccess && ak.type == cudaMemoryTypeHost;
    if (direct && desc) direct = cudaPointerGetAttributes(&ad, desc) == cudaSuccess && ad.type == cudaMemoryTypeHost;
    cudaGetLastError();
    sgs_keypoint* hk = direct ? kps : ex->h_kps;
    uint8_t* hd = direct ? desc : ex->h_desc;
    SGS_CUDA_TRY(cudaMemcpyAsync(ex->h_count, ex->d_out_count, sizeof(int32_t) * nframes, cudaMemcpyDeviceToHost, st));
    SGS_CUDA_TRY(cudaMemcpyAsync(ex->h_error, ex->d_error, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SGS_CUDA_TRY(cudaMemcpyAsync(hk, ex->d_out_kps, sizeof(sgs_keypoint) * K * nframes, cudaMemcpyDeviceToHost, st));
    if (desc) SGS_CUDA_TRY(cudaMemcpyAsync(hd, ex->d_out_desc, 32 * K * nframes, cudaMemcpyDeviceToHost, st));
    SGS_CUDA_TRY(cudaStreamSynchronize(st));
    if (*ex->h_error) { set_error("device capacity overflow (code %d)", *ex->h_error); cudaMemsetAsync(ex->d_error, 0, 4, st); return SGS_ERR_CAPACITY; }
    for (int f = 0; f < nframes; ++f) {
        const int c = ex->h_count[f];
        n[f] = c;
        if (c > cap) { set_error("frame %d has %d keypoints, caller capacity is %d", f, c, cap); return SGS_ERR_CAPACITY; }
        if (!direct) {
            std::memcpy(kps + (size_t)f * cap, ex->h_kps + (size_t)f * K, sizeof(sgs_keypoint) * c);
            if (desc) std::memcpy(desc + (size_t)f * cap * 32, ex->h_desc + (size_t)f * K * 32, (size_t)32 * c);
        }
    }
    return SGS_OK;
}

SGS_API int sgs_extract_batch(sgs_extractor* ex, const uint8_t* gray, int nframes, size_t frame_stride, int pitch, sgs_keypoint* kps,
                              uint8_t* desc, int cap, int* n) {
    const bool no_fetch = ex && !kps && !desc && !n && gray;      // upload + kernels only: the results stay on the device (sgs_extractor_results_device)
    if (!ex || (!n && !no_fetch)) return fail_invalid("sgs_extract_batch: NULL argument");
    if (nframes < 0 || nframes > ex->max_batch) return fail_invalid("sgs_extract_batch: nframes outside [0,max_batch]");
    if (nframes == 0) return SGS_OK;
    if (!gray) { for (int f = 0; f < nframes; ++f) n[f] = 0; return SGS_OK; }  // empty image: ORBextractor.cc:1048
    if (!kps && !no_fetch) return fail_invalid("sgs_extract_batch: NULL output");    // desc == NULL: keypoints only
    const OrbPlan& PL = ex->plan;
    if (pitch < PL.width || frame_stride < (size_t)pitch * PL.height) return fail_invalid("sgs_extract_batch: pitch/frame_stride too small");
    SGS_CUDA_TRY(cudaSetDevice(ex->device));
    cudaStream_t st = ex->stream;
    const LevelGeom& g0 = PL.lv[0];
    // pinned caller memory is copied straight to the device; pageable memory goes through the pinned staging buffer
    cudaPointerAttributes attr;
    const bool pinned = cudaPointerGetAttributes(&attr, gray) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (pinned && nframes >= 64) {
        // large pinned batches: the frames go up in chunks on the copy stream while the kernels of the previous chunk run
        const int nchunks = nframes >= 256 ? 4 : 2;
        const int per = (nframes + nchunks - 1) / nchunks;
        SGS_CUDA_TRY(cudaEventRecord(ex->chunk_done, st));                     // work already queued on st may still read the staging buffer
        SGS_CUDA_TRY(cudaStreamWaitEvent(ex->copy_stream, ex->chunk_done, 0));
        for (int c = 0, f0 = 0; f0 < nframes; ++c, f0 += per) {
            const int nf = std::min(per, nframes - f0);
            if (frame_stride == (size_t)pitch * PL.height) {
                SGS_CUDA_TRY(cudaMemcpy2DAsync(ex->d_pyr + (size_t)f0 * g0.frame_stride, g0.pitch, gray + (size_t)f0 * frame_stride, pitch, PL.width,
                                               (size_t)PL.height * nf, cudaMemcpyHostToDevice, ex->copy_stream));
            } else {
                for (int f = f0; f < f0 + nf; ++f)
                    SGS_CUDA_TRY(cudaMemcpy2DAsync(ex->d_pyr + (size_t)f * g0.frame_stride, g0.pitch, gray + (size_t)f * frame_stride, pitch, PL.width, PL.height,
                                                   cudaMemcpyHostToDevice, ex->copy_stream));
            }
            SGS_CUDA_TRY(cudaEventRecord(ex->chunk_ev[c], ex->copy_stream));
            SGS_CUDA_TRY(cudaStreamWaitEvent(st, ex->chunk_ev[c], 0));
            const int rc = enqueue(ex, ex->d_pyr, g0.pitch, g0.frame_stride, nf, st, f0, nframes, false);
            if (rc != SGS_OK) return rc;
        }
        ex->last_level0_external = false;
        return no_fetch ? SGS_OK : sgs_extractor_fetch(ex, nframes, kps, desc, cap, n, st);
    }
    if (pinned) {
        if (frame_stride == (size_t)pitch * PL.height) {
            SGS_CUDA_TRY(cudaMemcpy2DAsync(ex->d_pyr, g0.pitch, gray, pitch, PL.width, (size_t)PL.height * nframes, cudaMemcpyHostToDevice, st));
        } else {
            for (int f = 0; f < nframes; ++f)
                SGS_CUDA_TRY(cudaMemcpy2DAsync(ex->d_pyr + (size_t)f * g0.frame_stride, g0.pitch, gray + (size_t)f * frame_stride, pitch, PL.width, PL.height, cudaMemcpyHostToDevice, st));
        }
    } else {
        for (int f = 0; f < nframes; ++f)
            for (int y = 0; y < PL.height; ++y)
                std::memcpy(ex->h_in + (size_t)f * g0.frame_stride + (size_t)y * g0.pitch, gray + (size_t)f * frame_stride + (size_t)y * pitch, PL.width);
        SGS_CUDA_TRY(cudaMemcpyAsync(ex->d_pyr, ex->h_in, (size_t)nframes * g0.frame_stride, cudaMemcpyHostToDevice, st));
    }
    ex->last_level0_external = false;
    int rc = enqueue(ex, ex->d_pyr, g0.pitch, g0.frame_stride, nframes, st);
    if (rc != SGS_OK) return rc;
    return no_fetch ? SGS_OK : sgs_extractor_fetch(ex, nframes, kps, desc, cap, n, st);
}

SGS_API void* sgs_extractor_stream(const sgs_extractor* ex) { return ex ? (void*)ex->stream : nullptr; }

SGS_API int sgs_extract(sgs_extractor* ex, const uint8_t* gray, int width, int height, int pitch, sgs_keypoint* kps, uint8_t* desc, int cap, int* n) {
    if (!ex || !n) return fail_invalid("sgs_extract: NULL argument");
    if (!gray || width == 0 || height == 0) { *n = 0; return SGS_OK; }
    if (width != ex->plan.width || height != ex->plan.height) return fail_invalid("sgs_extract: image size differs from the handle's geometry");
    return sgs_extract_batch(ex, gray, 1, (size_t)pitch * height, pitch, kps, desc, cap, n);
}

SGS_API int sgs_memcpy_d2h(void* dst, const void* d_src, size_t bytes) {   // harness helper: plain synchronous device -> host copy
    if (!dst || !d_src) return fail_invalid("sgs_memcpy_d2h: NULL");
    SGS_CUDA_TRY(cudaMemcpy(dst, d_src, bytes, cudaMemcpyDeviceToHost));
    return SGS_OK;
}

SGS_API int sgs_extractor_level0_device(const sgs_extractor* ex, const uint8_t** d_frames, int* pitch, size_t* frame_stride) {
    if (!ex) return fail_invalid("sgs_extractor_level0_device: NULL handle");
    if (d_frames) *d_frames = ex->d_pyr;
    if (pitch) *pitch = ex->plan.lv[0].pitch;
    if (frame_stride) *frame_stride = (size_t)ex->plan.lv[0].frame_stride;
    return SGS_OK;
}

SGS_API int sgs_extractor_read_level(sgs_extractor* ex, int frame, int level, int blurred, uint8_t* out, int out_pitch) {
    if (!ex || !out || level < 0 || level >= ex->plan.nlevels || frame < 0 || frame >= ex->last_nframes) return fail_invalid("sgs_extractor_read_level: bad argument");
    if (level == 0 && !blurred && ex->last_level0_external) return fail_invalid("sgs_extractor_read_level: level 0 aliases the caller's buffer");
    SGS_CUDA_TRY(cudaSetDevice(ex->device));
    const LevelGeom& g = ex->plan.lv[level];
    const uint8_t* base = (blurred ? ex->d_blur : ex->d_pyr) + ex->lvl_off[level] + (int64_t)frame * g.frame_stride;
    SGS_CUDA_TRY(cudaStreamSynchronize(ex->stream));
    SGS_CUDA_TRY(cudaMemcpy2D(out, out_pitch, base, g.pitch, g.w, g.h, cudaMemcpyDeviceToHost));
    return SGS_OK;
}

SGS_API int sgs_extractor_read_candidates(sgs_extractor* ex, int frame, int level, int32_t* xyscore, int cap, int* n) {
    if (!ex || !n || level < 0 || level >= ex->plan.nlevels || frame < 0 || frame >= ex->last_nframes) return fail_invalid("sgs_extractor_read_candidates: bad argument");
    SGS_CUDA_TRY(cudaSetDevice(ex->device));
    SGS_CUDA_TRY(cudaStreamSynchronize(ex->stream));
    int32_t cnt = 0;
    SGS_CUDA_TRY(cudaMemcpy(&cnt, ex->d_cand_count + frame * ex->plan.nlevels + level, 4, cudaMemcpyDeviceToHost));
    *n = cnt;
    if (cnt > cap || !xyscore) { set_error("candidate buffer too small: need %d", cnt); return SGS_ERR_CAPACITY; }
    std::vector<uint32_t> h(cnt > 0 ? cnt : 1);
    SGS_CUDA_TRY(cudaMemcpy(h.data(), ex->d_cand + (int64_t)frame * ex->plan.cand_per_frame + ex->plan.lv[level].cand_off, sizeof(uint32_t) * cnt, cudaMemcpyDeviceToHost));
    for (int i = 0; i < cnt; ++i) { xyscore[3 * i] = qt_x(h[i]); xyscore[3 * i + 1] = qt_y(h[i]); xyscore[3 * i + 2] = qt_score(h[i]); }
    return SGS_OK;
}

}  // extern "C"
