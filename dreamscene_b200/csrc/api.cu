// C ABI (include/b200gsr.h, include/b200gsr_scene.h, include/b200gsr_step.h, include/b200gsr_loss.h): argument
// validation, buffer layouts, launch sequencing.
#include "common.cuh"
#include "../../include/b200gsr_step.h"
#include "../../include/b200gsr_loss.h"
#include "../../include/b200gsr_frozen.h"
#include "../../include/b200gsr_stats.h"
#include "../../include/b200gsr_reserve.h"
#include "../../include/b200gsr_frames.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#ifndef B200GSR_NO_NVTX
#include <nvtx3/nvToolsExt.h>   // header-only; a no-op unless a profiler is attached
#define GSR_RANGE_PUSH(name) nvtxRangePushA(name)
#define GSR_RANGE_POP() nvtxRangePop()
#else
#define GSR_RANGE_PUSH(name) ((void)0)
#define GSR_RANGE_POP() ((void)0)
#endif

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return B200GSR_OK;
    return fail(B200GSR_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

// ---- optional per-stage timing (process-wide, not thread-safe; used by bench.py only) ----------
enum { kFwdEvents = 6, kBwdEvents = 3 };
struct Prof {
    int max_calls = 0;
    int nfwd = 0, nbwd = 0;
    cudaEvent_t* fwd = nullptr;   // [max_calls][kFwdEvents]
    cudaEvent_t* bwd = nullptr;   // [max_calls][kBwdEvents]
} g_prof;

void prof_mark_fwd(int k, cudaStream_t s) {
    if (g_prof.max_calls > 0 && g_prof.nfwd < g_prof.max_calls)
        cudaEventRecord(g_prof.fwd[g_prof.nfwd * kFwdEvents + k], s);
}
void prof_mark_bwd(int k, cudaStream_t s) {
    if (g_prof.max_calls > 0 && g_prof.nbwd < g_prof.max_calls)
        cudaEventRecord(g_prof.bwd[g_prof.nbwd * kBwdEvents + k], s);
}

// ---- per-device state, created lazily under a mutex and never destroyed: SM count + a forked
// stream that lets the two tile-sort size classes run concurrently.
struct DeviceState {
    bool ready = false;
    int num_sms = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
};
DeviceState g_dev[64];
unsigned long long* g_stats = nullptr;   // b200gsr_debug_counters (process-wide, diagnostics only)
std::mutex g_dev_mutex;

// Returns nullptr only if the device ordinal is out of range or CUDA itself fails.
DeviceState* device_state() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    DeviceState& s = g_dev[dev];
    if (s.ready) return &s;                       // written once under the mutex
    std::lock_guard<std::mutex> lock(g_dev_mutex);
    if (s.ready) return &s;
    int nsm = 132;
    if (cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && nsm > 0) s.num_sms = nsm;
    // the side stream is optional: without it the two sort kernels simply run back to back
    cudaStream_t st = nullptr;
    cudaEvent_t ef = nullptr, ej = nullptr;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess &&
        cudaEventCreateWithFlags(&ef, cudaEventDisableTiming) == cudaSuccess &&
        cudaEventCreateWithFlags(&ej, cudaEventDisableTiming) == cudaSuccess) {
        s.stream = st; s.fork = ef; s.join = ej;
    } else {
        if (ef) cudaEventDestroy(ef);
        if (ej) cudaEventDestroy(ej);
        if (st) cudaStreamDestroy(st);
        cudaGetLastError();   // clear the non-sticky creation error
    }
    s.ready = true;
    return &s;
}

// The checks the score pass shares with a full forward: the image size, and exactly one shape input per Gaussian.
// `view` < 0 leaves the view out of the messages (single-view entry points).
int check_size(const b200gsr_params& p, int view) {
    if (p.P < 0 || p.image_height < 0 || p.image_width < 0)
        return view < 0 ? fail(B200GSR_ERR_BAD_ARG, "negative size") : fail(B200GSR_ERR_BAD_ARG, "view %d: negative size", view);
    if (p.image_height > 65535 * 16 || p.image_width > 65535 * 16)
        return fail(B200GSR_ERR_UNSUPPORTED, "image larger than 65535 tiles per axis");
    return B200GSR_OK;
}

int check_shape_inputs(const float* scales, const float* rots, const float* cov3d) {
    const bool has_sr = scales != nullptr || rots != nullptr;
    if (((scales == nullptr || rots == nullptr) && cov3d == nullptr) || (has_sr && cov3d != nullptr))
        return fail(B200GSR_ERR_BAD_ARG, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    return B200GSR_OK;
}

int validate_inputs(const b200gsr_params* p, const float* means3D, const float* shs,
                    const float* colors, const float* opac, const float* scales,
                    const float* rots, const float* cov3d) {
    if (!p) return fail(B200GSR_ERR_BAD_ARG, "params is null");
    int rc = check_size(*p, -1);
    if (rc) return rc;
    if (!p->bg || !p->viewmatrix || !p->projmatrix || !p->campos)
        return fail(B200GSR_ERR_BAD_ARG, "bg/viewmatrix/projmatrix/campos must be device pointers");
    if (p->P > 0) {
        if (!means3D || !opac) return fail(B200GSR_ERR_BAD_ARG, "means3D/opacities are required");
        if ((shs != nullptr) == (colors != nullptr))
            return fail(B200GSR_ERR_BAD_ARG, "Please provide excatly one of either SHs or precomputed colors!");
        if ((rc = check_shape_inputs(scales, rots, cov3d))) return rc;
        if (shs) {
            if (p->sh_degree < 0 || p->sh_degree > 3)
                return fail(B200GSR_ERR_UNSUPPORTED, "sh_degree %d not in 0..3", p->sh_degree);
            if (p->M < (p->sh_degree + 1) * (p->sh_degree + 1) || p->M > 16)
                return fail(B200GSR_ERR_BAD_ARG, "M=%d inconsistent with sh_degree=%d (need (deg+1)^2 <= M <= 16)",
                            p->M, p->sh_degree);
        }
    }
    return B200GSR_OK;
}

// The deterministic accumulators (GsrDetLayout) follow everything b200gsr_saved_layout describes, so that layout's
// offsets and its total without B200GSR_SAVED_DETERMINISTIC stay what they always were.
GsrDetLayout det_layout(int32_t P, size_t base, bool with_backward) {
    GsrDetLayout d{};
    size_t off = base;
    if (with_backward) {
        d.dmax = off; off = align_up(off + (size_t)P * GSR_DET_COMPONENTS * sizeof(uint32_t));
        d.dfx = off;  off = align_up(off + (size_t)P * GSR_DET_COMPONENTS * sizeof(unsigned long long));
    }
    d.score_fx = off; off = align_up(off + (size_t)P * sizeof(unsigned long long));
    d.total = off;
    return d;
}

// Deterministic sums have overflow headroom for GSR_DET_MAX_VIEW_TILES tiles per view (common.cuh).
int check_det_size(int32_t H, int32_t W) {
    if ((long long)gsr_grid(H, W).ntiles > GSR_DET_MAX_VIEW_TILES)
        return fail(B200GSR_ERR_UNSUPPORTED, "deterministic mode supports at most %d 16x16 tiles per view (8192x8192); "
                    "the image is %dx%d", GSR_DET_MAX_VIEW_TILES, W, H);
    return B200GSR_OK;
}

// The three forwards differ only in their validation, in the height their layouts describe, and in the two
// per-view / per-tile stages:
//   kImage  b200gsr_forward: one view; the layouts describe the image itself; records the profiling events.
//   kViews  b200gsr_forward_views: the layouts describe the stacked image (even for B = 1); no profiling events.
//   kScore  b200gsr_score_views: stacked; geometry-only projection and score-only compositing into the caller's
//           accumulator, which holds the deterministic sum itself, so `saved` carries no deterministic state.
//   kScene  b200gsr_forward_scene: stacked; the projection reads the raw leaves of `scene` (in == null); records the
//           profiling events.
enum class Pass { kImage, kViews, kScore, kScene };

// Everything a forward does after its entry point's validation, for B views stacked vertically.  Every size and
// workspace refusal comes before device_state(), the first CUDA call.  `score` is the float [B*P] score of a
// render, or the [P] accumulator of the score pass.
int run_forward(Pass pass, int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in, float* out_color,
                float* out_depth_alpha, int32_t* radii, void* score, void* scratch, size_t scratch_bytes, void* saved,
                size_t saved_bytes, uint64_t max_pairs, uint32_t flags, uint32_t* host_notify, uint32_t notify_seq,
                void* stream, const GsrScene* scene = nullptr) {
    const bool score_pass = pass == Pass::kScore;
    const int P = prm[0].P, H = prm[0].image_height, W = prm[0].image_width;
    const GsrTileGrid g1 = gsr_grid(H, W);
    const int Hs = pass == Pass::kImage ? H : B * g1.gy * GSR_TILE;
    if (score_pass) flags |= B200GSR_FWD_NO_BACKWARD;
    GsrFwdArgs a{};
    const int with_bwd = (flags & B200GSR_FWD_NO_BACKWARD) ? 0 : 1;
    a.det = (flags & B200GSR_FWD_DETERMINISTIC) != 0;
    int rc;
    if (a.det && (rc = check_det_size(H, W))) return rc;
    if (a.det && score_pass && (long long)B * H * W > B200GSR_SCORE_DET_MAX_PIXELS)
        return fail(B200GSR_ERR_UNSUPPORTED, "deterministic score: %d views of %dx%d exceed 2^26 pixels per accumulator", B, W, H);
    if ((rc = b200gsr_scratch_layout_query(B * P, Hs, W, max_pairs, &a.sl))) return rc;
    if ((rc = b200gsr_saved_layout_query(B * P, Hs, W, max_pairs, with_bwd, &a.vl))) return rc;
    a.dl = det_layout(B * P, a.vl.total, with_bwd != 0);
    const size_t saved_need = a.det && !score_pass ? a.dl.total : a.vl.total;
    if (scratch_bytes < a.sl.total || saved_bytes < saved_need)
        return fail(B200GSR_ERR_WORKSPACE, "workspace too small: scratch %zu < %zu or saved %zu < %zu",
                    scratch_bytes, a.sl.total, saved_bytes, saved_need);
    DeviceState* ds = device_state();
    if (!ds) return fail(B200GSR_ERR_CUDA, "cannot query the current CUDA device");
    a.out_color = out_color; a.out_depth_alpha = out_depth_alpha; a.radii = radii;
    a.score = score_pass ? nullptr : static_cast<float*>(score);
    a.scratch = static_cast<uint8_t*>(scratch); a.saved = static_cast<uint8_t*>(saved);
    a.max_pairs = (uint32_t)max_pairs;
    a.host_notify = host_notify; a.notify_seq = notify_seq;
    a.flags = flags; a.num_sms = ds->num_sms; a.stats = score_pass ? nullptr : g_stats;
    a.num_views = B; a.P_view = P; a.gy_view = g1.gy;
    a.stream = static_cast<cudaStream_t>(stream);
    a.scene = scene;
    const bool profile = pass != Pass::kViews;

    // The counters at the start of scratch must be zero before the count kernel runs.  On the main path
    // (multisplit binning, P > 0) the projection prologue zeroes them; only the large-grid fallback (the
    // projection itself counts with global atomics) and the P == 0 case need a memset node.
    const int ntiles = g1.gx * g1.gy * B;
    if (!gsr_use_multisplit(ntiles) || P == 0) {
        const size_t nbytes = gsr_counter_words(a.sl, ntiles) * sizeof(uint32_t);
        if ((rc = check_cuda(cudaMemsetAsync(a.scratch, 0, nbytes, a.stream), "memset"))) return rc;
    }
    if (profile) prof_mark_fwd(0, a.stream);
    GSR_RANGE_PUSH("b200gsr.project+count");
    for (int v = 0; v < B && !rc; ++v) {
        a.prm = prm[v]; a.view = v;
        if (in) {
            a.means3D = in[v].means3D; a.shs = in[v].shs; a.colors = in[v].colors_precomp; a.opac = in[v].opacities;
            a.scales = in[v].scales; a.rots = in[v].rotations; a.cov3d = in[v].cov3D_precomp;
        }
        rc = check_cuda(gsr_launch_project(a, score_pass), score_pass ? "project_geo" : "project_sh");
    }
    a.prm = prm[0]; a.view = 0;     // per-view constants are not used past this point (bg is indexed by tile row)
    if (!rc) rc = check_cuda(gsr_launch_count(a), "tile_count");
    GSR_RANGE_POP();
    if (rc) return rc;
    if (profile) prof_mark_fwd(1, a.stream);
    GSR_RANGE_PUSH("b200gsr.scan_order");
    rc = check_cuda(gsr_launch_scan(a), "scan_order");
    GSR_RANGE_POP();
    if (rc) return rc;
    if (profile) prof_mark_fwd(2, a.stream);
    GSR_RANGE_PUSH("b200gsr.scatter");
    rc = check_cuda(gsr_launch_scatter(a), "scatter");
    GSR_RANGE_POP();
    if (rc) return rc;
    if (profile) prof_mark_fwd(3, a.stream);
    GSR_RANGE_PUSH("b200gsr.tile_sort");
    rc = check_cuda(gsr_launch_sort(a, ds->stream, ds->fork, ds->join), "tile_sort");
    GSR_RANGE_POP();
    if (rc) return rc;
    if (profile) prof_mark_fwd(4, a.stream);
    GSR_RANGE_PUSH("b200gsr.composite");
    rc = score_pass ? check_cuda(gsr_launch_composite_score(a, score), "composite_score")
                    : check_cuda(gsr_launch_composite_fwd(a), "composite_fwd");
    GSR_RANGE_POP();
    if (rc) return rc;
    if (profile) {
        prof_mark_fwd(5, a.stream);
        if (g_prof.max_calls > 0 && g_prof.nfwd < g_prof.max_calls) ++g_prof.nfwd;
    }
    return B200GSR_OK;
}

// The setup both backward entry points share after their validation: the saved layout of the forward (`stacked`
// as in run_forward's kViews) and its size check, then every field of `a` but the per-view and per-range ones.
int setup_backward(bool stacked, int32_t B, const b200gsr_params* prm, const int32_t* radii,
                   const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha, void* saved,
                   size_t saved_bytes, uint64_t max_pairs, bool det, void* stream, GsrBwdArgs& a) {
    const int P = prm[0].P, H = prm[0].image_height, W = prm[0].image_width;
    const GsrTileGrid g1 = gsr_grid(H, W);
    a = GsrBwdArgs{};
    a.det = det;
    int rc;
    if (a.det && (rc = check_det_size(H, W))) return rc;
    if ((rc = b200gsr_saved_layout_query(B * P, stacked ? B * g1.gy * GSR_TILE : H, W, max_pairs, 1, &a.vl))) return rc;
    a.dl = det_layout(B * P, a.vl.total, true);
    const size_t saved_need = a.det ? a.dl.total : a.vl.total;
    if (saved_bytes < saved_need)
        return fail(B200GSR_ERR_WORKSPACE, "saved buffer too small for backward: %zu < %zu (was the forward "
                    "run with B200GSR_FWD_NO_BACKWARD, or without B200GSR_FWD_DETERMINISTIC?)", saved_bytes, saved_need);
    DeviceState* ds = device_state();
    if (!ds) return fail(B200GSR_ERR_CUDA, "cannot query the current CUDA device");
    a.prm = prm[0];
    a.radii = radii; a.out_depth_alpha = out_depth_alpha; a.dL_dcolor = dL_dcolor; a.dL_ddepth_alpha = dL_ddepth_alpha;
    a.saved = static_cast<uint8_t*>(saved); a.max_pairs = (uint32_t)max_pairs;
    a.num_sms = ds->num_sms; a.stats = g_stats;
    a.num_views = B; a.P_view = P; a.gy_view = g1.gy;
    a.stream = static_cast<cudaStream_t>(stream);
    return B200GSR_OK;
}

void set_view_inputs(GsrBwdArgs& a, const b200gsr_view_inputs& in) {
    a.means3D = in.means3D; a.shs = in.shs; a.colors = in.colors_precomp; a.opac = in.opacities;
    a.scales = in.scales; a.rots = in.rotations; a.cov3d = in.cov3D_precomp;
}

bool has_view_grads(const b200gsr_view_inputs& in, const b200gsr_view_grads& o) {
    return o.d_means3D && o.d_means2D && o.d_opacities && (!in.shs || o.d_shs) && (!in.colors_precomp || o.d_colors) &&
           (!in.cov3D_precomp || o.d_cov3D) && (in.cov3D_precomp || (o.d_scales && o.d_rotations));
}

}  // namespace

extern "C" {

int b200gsr_version(void) { return B200GSR_VERSION; }

const char* b200gsr_last_error(void) { return g_err; }

int b200gsr_saved_layout_query(int32_t P, int32_t H, int32_t W, uint64_t max_pairs,
                               int32_t with_backward, b200gsr_saved_layout* out) {
    if (!out || P < 0 || H < 0 || W < 0) return fail(B200GSR_ERR_BAD_ARG, "bad layout query");
    if (max_pairs > 0xfffffff0ull) return fail(B200GSR_ERR_UNSUPPORTED, "max_pairs must fit in 32 bits");
    const bool det = (with_backward & B200GSR_SAVED_DETERMINISTIC) != 0;
    with_backward &= ~B200GSR_SAVED_DETERMINISTIC;
    const GsrTileGrid g = gsr_grid(H, W);
    size_t off = 0;
    out->header = off;      off = align_up(off + GSR_H_WORDS * sizeof(uint32_t));
    out->tile_start = off;  off = align_up(off + ((size_t)g.ntiles + 1) * sizeof(uint32_t));
    out->work_order = off;  off = align_up(off + (size_t)g.ntiles * sizeof(uint32_t));
    out->n_contrib = off;   off = align_up(off + (size_t)H * W * sizeof(uint32_t));
    out->keys = off;        off = align_up(off + ((size_t)max_pairs + 2) * sizeof(uint64_t));
    out->geom = off;        off = align_up(off + (size_t)P * sizeof(GsrRec));
    out->dgeom = off;       off = align_up(off + (with_backward ? (size_t)P * 12 * sizeof(float) : 0));
    out->bwd_items = off;   off = align_up(off + (with_backward ? (size_t)GSR_BWD_CLASSES * g.ntiles * 8 * sizeof(uint32_t) : 0));
    out->total = det ? det_layout(P, off, with_backward != 0).total : off;
    return B200GSR_OK;
}

int b200gsr_scratch_layout_query(int32_t P, int32_t H, int32_t W, uint64_t max_pairs,
                                 b200gsr_scratch_layout* out) {
    if (!out || P < 0 || H < 0 || W < 0) return fail(B200GSR_ERR_BAD_ARG, "bad layout query");
    if (max_pairs > 0xfffffff0ull) return fail(B200GSR_ERR_UNSUPPORTED, "max_pairs must fit in 32 bits");
    const GsrTileGrid g = gsr_grid(H, W);
    size_t off = 0;
    out->counters = off;    off = align_up(off + GSR_NCOUNTERS * sizeof(uint32_t));
    out->tile_count = off;  off = align_up(off + (size_t)GSR_COPIES * g.ntiles * sizeof(uint32_t));
    out->tile_cursor = off; off = align_up(off + (size_t)GSR_COPIES * g.ntiles * sizeof(uint32_t));
    out->rectdepth = off;   off = align_up(off + (size_t)P * sizeof(uint4));
    out->ms_hist = off;
    if (gsr_use_multisplit(g.ntiles)) {   // per-CTA tile histograms, then the padded key buffer (common.cuh)
        off = gsr_pad_keys_offset(*out, P, g.ntiles);
        off = align_up(off + (size_t)gsr_pad_key_capacity(max_pairs, P, g.ntiles) * sizeof(unsigned long long));
    }
    out->total = off;
    return B200GSR_OK;
}

int b200gsr_forward(const b200gsr_params* prm, const float* means3D, const float* shs,
                    const float* colors_precomp, const float* opacities, const float* scales,
                    const float* rotations, const float* cov3D_precomp, float* out_color,
                    float* out_depth_alpha, int32_t* radii, float* score, void* scratch,
                    size_t scratch_bytes, void* saved, size_t saved_bytes, uint64_t max_pairs,
                    uint32_t flags, uint32_t* host_notify, uint32_t notify_seq, void* stream) {
    int rc = validate_inputs(prm, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp);
    if (rc) return rc;
    if (!out_color || !out_depth_alpha || (prm->P > 0 && !radii) || !scratch || !saved)
        return fail(B200GSR_ERR_BAD_ARG, "null output/workspace pointer");
    if (prm->score_flag && prm->P > 0 && !score)
        return fail(B200GSR_ERR_BAD_ARG, "score_flag set but score buffer is null");
    const b200gsr_view_inputs in = {means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp};
    return run_forward(Pass::kImage, 1, prm, &in, out_color, out_depth_alpha, radii, score, scratch, scratch_bytes, saved,
                       saved_bytes, max_pairs, flags, host_notify, notify_seq, stream);
}

int b200gsr_backward_ex(const b200gsr_params* prm, const float* means3D, const float* shs,
                     const float* colors_precomp, const float* opacities, const float* scales,
                     const float* rotations, const float* cov3D_precomp, const int32_t* radii,
                     const float* out_depth_alpha, const float* dL_dcolor,
                     const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                     void* /*scratch*/, size_t /*scratch_bytes*/, uint64_t max_pairs, float* d_means3D,
                     float* d_means2D, float* d_shs, float* d_colors, float* d_opacities,
                     float* d_scales, float* d_rotations, float* d_cov3D, uint32_t stages,
                     int32_t g_begin, int32_t g_end, int32_t dsh_coefs, void* stream) {
    int rc = validate_inputs(prm, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp);
    if (rc) return rc;
    if (prm->P == 0) return B200GSR_OK;
    if (g_begin < 0 || g_end > prm->P || g_begin > g_end || (g_begin % 128) != 0)
        return fail(B200GSR_ERR_BAD_ARG, "bad Gaussian range [%d, %d): need 0 <= begin <= end <= P, begin %% 128 == 0", g_begin, g_end);
    if (shs && dsh_coefs != 0 && dsh_coefs != -1 &&
        (dsh_coefs < (prm->sh_degree + 1) * (prm->sh_degree + 1) || dsh_coefs > prm->M))
        return fail(B200GSR_ERR_BAD_ARG, "dsh_coefs=%d must be 0, -1 or in [(sh_degree+1)^2, M]", dsh_coefs);
    if (!shs && dsh_coefs < 0) return fail(B200GSR_ERR_BAD_ARG, "dsh_coefs=-1 (factored SH gradient) needs shs");
    if (!radii || !out_depth_alpha || !dL_dcolor || !dL_ddepth_alpha || !saved)
        return fail(B200GSR_ERR_BAD_ARG, "null saved-state/gradient pointer");
    const b200gsr_view_inputs in = {means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp};
    const b200gsr_view_grads o = {d_means3D, d_means2D, d_shs, d_colors, d_opacities, d_scales, d_rotations, d_cov3D, 0};
    if (!has_view_grads(in, o)) return fail(B200GSR_ERR_BAD_ARG, "null gradient output pointer");
    GsrBwdArgs a;
    if ((rc = setup_backward(false, 1, prm, radii, out_depth_alpha, dL_dcolor, dL_ddepth_alpha, saved, saved_bytes,
                             max_pairs, (stages & B200GSR_BWD_DETERMINISTIC) != 0, stream, a)))
        return rc;
    set_view_inputs(a, in);
    a.d_means3D = d_means3D; a.d_means2D = d_means2D; a.d_shs = d_shs; a.d_colors = d_colors;
    a.d_opac = d_opacities; a.d_scales = d_scales; a.d_rots = d_rotations; a.d_cov3d = d_cov3D;
    a.g_begin = g_begin; a.g_end = g_end; a.dsh_coefs = dsh_coefs;

    // no memsets: the work-queue counters and the gradient accumulators live in `saved`, zeroed by
    // the forward and restored to zero by project_bwd
    const bool whole = (stages & B200GSR_BWD_COMPOSITE) && (stages & B200GSR_BWD_PROJECT) && g_begin == 0 && g_end == prm->P;
    if (stages & B200GSR_BWD_COMPOSITE) {
        if (whole) prof_mark_bwd(0, a.stream);
        GSR_RANGE_PUSH("b200gsr.composite_bwd");
        rc = check_cuda(gsr_launch_composite_bwd(a), "composite_bwd");
        GSR_RANGE_POP();
        if (rc) return rc;
    }
    if (stages & B200GSR_BWD_PROJECT) {
        if (whole) prof_mark_bwd(1, a.stream);
        GSR_RANGE_PUSH("b200gsr.project_bwd");
        rc = check_cuda(gsr_launch_project_bwd(a), "project_bwd");
        GSR_RANGE_POP();
        if (rc) return rc;
    }
    if (whole) {
        prof_mark_bwd(2, a.stream);
        if (g_prof.max_calls > 0 && g_prof.nbwd < g_prof.max_calls) ++g_prof.nbwd;
    }
    return B200GSR_OK;
}

int b200gsr_backward(const b200gsr_params* prm, const float* means3D, const float* shs,
                     const float* colors_precomp, const float* opacities, const float* scales,
                     const float* rotations, const float* cov3D_precomp, const int32_t* radii,
                     const float* out_depth_alpha, const float* dL_dcolor,
                     const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                     void* scratch, size_t scratch_bytes, uint64_t max_pairs, float* d_means3D,
                     float* d_means2D, float* d_shs, float* d_colors, float* d_opacities,
                     float* d_scales, float* d_rotations, float* d_cov3D, void* stream) {
    return b200gsr_backward_ex(prm, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, radii,
                               out_depth_alpha, dL_dcolor, dL_ddepth_alpha, saved, saved_bytes, scratch, scratch_bytes,
                               max_pairs, d_means3D, d_means2D, d_shs, d_colors, d_opacities, d_scales, d_rotations,
                               d_cov3D, B200GSR_BWD_COMPOSITE | B200GSR_BWD_PROJECT, 0, prm ? prm->P : 0, 0, stream);
}

// ---------------------------------------------------------------------------------------------
// Multi-view entry points (SURVEY.md 8 f1): B views of the same image size in ONE binning / sort /
// composite pass.  The views are stacked vertically into an image of B * gy tile rows and view v's
// Gaussians become the virtual Gaussians [v*P, (v+1)*P): only the two per-Gaussian stages run per view
// (each with its own camera and, if the caller wishes, its own parameter tensors).
// ---------------------------------------------------------------------------------------------
static int check_views(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in) {
    if (B < 1 || B > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_UNSUPPORTED, "number of views %d not in 1..%d", B, B200GSR_MAX_VIEWS);
    if (!prm || !in) return fail(B200GSR_ERR_BAD_ARG, "null view array");
    for (int v = 0; v < B; ++v) {
        int rc = validate_inputs(&prm[v], in[v].means3D, in[v].shs, in[v].colors_precomp, in[v].opacities, in[v].scales,
                                 in[v].rotations, in[v].cov3D_precomp);
        if (rc) return rc;
        if (prm[v].P != prm[0].P || prm[v].M != prm[0].M || prm[v].image_height != prm[0].image_height ||
            prm[v].image_width != prm[0].image_width || prm[v].score_flag != prm[0].score_flag)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: P, M, image size and score_flag must equal view 0's", v);
        if (prm[v].bg != prm[0].bg + 3 * v)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: backgrounds must be one contiguous device array [B,3] (prm[v].bg = prm[0].bg + 3 v)", v);
        if ((in[v].shs != nullptr) != (in[0].shs != nullptr) || (in[v].cov3D_precomp != nullptr) != (in[0].cov3D_precomp != nullptr))
            return fail(B200GSR_ERR_BAD_ARG, "view %d: all views must use the same input kinds", v);
    }
    if ((long long)B * prm[0].P > 0x3fffffffLL) return fail(B200GSR_ERR_UNSUPPORTED, "B * P too large");
    return B200GSR_OK;
}

int b200gsr_views_geometry(int32_t B, int32_t H, int32_t W, int32_t* stacked_height) {
    if (B < 1 || H < 0 || W < 0 || !stacked_height) return fail(B200GSR_ERR_BAD_ARG, "bad views_geometry arguments");
    *stacked_height = B * gsr_grid(H, W).gy * GSR_TILE;
    return B200GSR_OK;
}

int b200gsr_forward_views(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in, float* out_color,
                          float* out_depth_alpha, int32_t* radii, float* score, void* scratch, size_t scratch_bytes,
                          void* saved, size_t saved_bytes, uint64_t max_pairs, uint32_t flags, uint32_t* host_notify,
                          uint32_t notify_seq, void* stream) {
    int rc = check_views(B, prm, in);
    if (rc) return rc;
    const int P = prm[0].P;
    if (!out_color || !out_depth_alpha || (P > 0 && !radii) || !scratch || !saved)
        return fail(B200GSR_ERR_BAD_ARG, "null output/workspace pointer");
    if (prm[0].score_flag && P > 0 && !score) return fail(B200GSR_ERR_BAD_ARG, "score_flag set but score buffer is null");
    return run_forward(Pass::kViews, B, prm, in, out_color, out_depth_alpha, radii, score, scratch, scratch_bytes, saved,
                       saved_bytes, max_pairs, flags, host_notify, notify_seq, stream);
}

int b200gsr_backward_views_ex(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in, const int32_t* radii,
                              const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha,
                              void* saved, size_t saved_bytes, uint64_t max_pairs, const b200gsr_view_grads* out,
                              uint32_t flags, void* stream) {
    int rc = check_views(B, prm, in);
    if (rc) return rc;
    const int P = prm[0].P;
    if (P == 0) return B200GSR_OK;
    if (!radii || !out_depth_alpha || !dL_dcolor || !dL_ddepth_alpha || !saved || !out)
        return fail(B200GSR_ERR_BAD_ARG, "null saved-state/gradient pointer");
    for (int v = 0; v < B; ++v)     // before any launch: composite_bwd consumes the work lists project_bwd needs
        if (!has_view_grads(in[v], out[v])) return fail(B200GSR_ERR_BAD_ARG, "view %d: null gradient output pointer", v);
    GsrBwdArgs a;
    if ((rc = setup_backward(true, B, prm, radii, out_depth_alpha, dL_dcolor, dL_ddepth_alpha, saved, saved_bytes,
                             max_pairs, (flags & B200GSR_BWD_DETERMINISTIC) != 0, stream, a)))
        return rc;
    set_view_inputs(a, in[0]);
    a.g_begin = 0; a.g_end = P;
    GSR_RANGE_PUSH("b200gsr.views.composite_bwd");
    rc = check_cuda(gsr_launch_composite_bwd(a), "composite_bwd");
    GSR_RANGE_POP();
    if (rc) return rc;
    GSR_RANGE_PUSH("b200gsr.views.project_bwd");
    for (int v = 0; v < B && !rc; ++v) {
        const b200gsr_view_grads& o = out[v];
        a.prm = prm[v]; a.view = v; a.accumulate = (int)o.accumulate;
        set_view_inputs(a, in[v]);
        a.d_means3D = o.d_means3D; a.d_means2D = o.d_means2D; a.d_shs = o.d_shs; a.d_colors = o.d_colors;
        a.d_opac = o.d_opacities; a.d_scales = o.d_scales; a.d_rots = o.d_rotations; a.d_cov3d = o.d_cov3D;
        rc = check_cuda(gsr_launch_project_bwd(a), "project_bwd");
    }
    GSR_RANGE_POP();
    return rc;
}

int b200gsr_backward_views(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in, const int32_t* radii,
                           const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha,
                           void* saved, size_t saved_bytes, uint64_t max_pairs, const b200gsr_view_grads* out,
                           void* stream) {
    return b200gsr_backward_views_ex(B, prm, in, radii, out_depth_alpha, dL_dcolor, dL_ddepth_alpha, saved, saved_bytes,
                                     max_pairs, out, 0u, stream);
}

// Score pass: only geometry and opacity are read, so the colour inputs validate_inputs insists on are not required.
static int check_score_views(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in) {
    if (B < 1 || B > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_UNSUPPORTED, "number of views %d not in 1..%d", B, B200GSR_MAX_VIEWS);
    if (!prm || !in) return fail(B200GSR_ERR_BAD_ARG, "null view array");
    for (int v = 0; v < B; ++v) {
        const b200gsr_params& p = prm[v];
        int rc = check_size(p, v);
        if (rc) return rc;
        if (!p.viewmatrix || !p.projmatrix || !p.campos)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: viewmatrix/projmatrix/campos must be device pointers", v);
        if (p.P != prm[0].P || p.image_height != prm[0].image_height || p.image_width != prm[0].image_width)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: P and image size must equal view 0's", v);
        if (p.P > 0) {
            const b200gsr_view_inputs& x = in[v];
            if (!x.means3D || !x.opacities) return fail(B200GSR_ERR_BAD_ARG, "view %d: means3D/opacities are required", v);
            if ((rc = check_shape_inputs(x.scales, x.rotations, x.cov3D_precomp))) return rc;
        }
    }
    if ((long long)B * prm[0].P > 0x3fffffffLL) return fail(B200GSR_ERR_UNSUPPORTED, "B * P too large");
    return B200GSR_OK;
}

int b200gsr_score_views(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in, void* score_acc,
                        void* scratch, size_t scratch_bytes, void* saved, size_t saved_bytes, uint64_t max_pairs,
                        uint32_t flags, uint32_t* host_notify, uint32_t notify_seq, void* stream) {
    int rc = check_score_views(B, prm, in);
    if (rc) return rc;
    if (flags & ~(B200GSR_FWD_NO_BACKWARD | B200GSR_FWD_DETERMINISTIC)) return fail(B200GSR_ERR_BAD_ARG, "unknown flags 0x%x", flags);
    if ((prm[0].P > 0 && !score_acc) || !scratch || !saved) return fail(B200GSR_ERR_BAD_ARG, "null accumulator/workspace pointer");
    return run_forward(Pass::kScore, B, prm, in, nullptr, nullptr, nullptr, score_acc, scratch, scratch_bytes, saved,
                       saved_bytes, max_pairs, flags, host_notify, notify_seq, stream);
}

int b200gsr_score_finish(int32_t P, const void* score_acc, float* score, uint32_t flags, void* stream) {
    if (P < 0 || (P > 0 && (!score_acc || !score))) return fail(B200GSR_ERR_BAD_ARG, "bad score_finish arguments");
    if (flags != B200GSR_FWD_DETERMINISTIC)
        return fail(B200GSR_ERR_BAD_ARG, "score_finish converts a deterministic (int64) accumulator: flags must be B200GSR_FWD_DETERMINISTIC");
    return check_cuda(gsr_launch_score_finish(P, static_cast<const unsigned long long*>(score_acc), score,
                                              static_cast<cudaStream_t>(stream)), "score_finish");
}

int b200gsr_profile_enable(int32_t max_calls) {
    for (int i = 0; i < g_prof.max_calls * kFwdEvents; ++i) cudaEventDestroy(g_prof.fwd[i]);
    for (int i = 0; i < g_prof.max_calls * kBwdEvents; ++i) cudaEventDestroy(g_prof.bwd[i]);
    delete[] g_prof.fwd; delete[] g_prof.bwd;
    g_prof = Prof();
    if (max_calls <= 0) return B200GSR_OK;
    g_prof.fwd = new cudaEvent_t[(size_t)max_calls * kFwdEvents];
    g_prof.bwd = new cudaEvent_t[(size_t)max_calls * kBwdEvents];
    for (int i = 0; i < max_calls * kFwdEvents; ++i)
        if (cudaEventCreate(&g_prof.fwd[i]) != cudaSuccess) return fail(B200GSR_ERR_CUDA, "cudaEventCreate");
    for (int i = 0; i < max_calls * kBwdEvents; ++i)
        if (cudaEventCreate(&g_prof.bwd[i]) != cudaSuccess) return fail(B200GSR_ERR_CUDA, "cudaEventCreate");
    g_prof.max_calls = max_calls;
    return B200GSR_OK;
}

int b200gsr_profile_counts(int32_t* n_forward, int32_t* n_backward) {
    if (n_forward) *n_forward = g_prof.nfwd;
    if (n_backward) *n_backward = g_prof.nbwd;
    return B200GSR_OK;
}

int b200gsr_profile_read(int32_t is_backward, int32_t call, float* ms) {
    if (!ms) return fail(B200GSR_ERR_BAD_ARG, "ms is null");
    const int n = is_backward ? g_prof.nbwd : g_prof.nfwd;
    if (call < 0 || call >= n) return fail(B200GSR_ERR_BAD_ARG, "profile call index %d out of range (%d)", call, n);
    const int ne = is_backward ? kBwdEvents : kFwdEvents;
    cudaEvent_t* ev = (is_backward ? g_prof.bwd : g_prof.fwd) + (size_t)call * ne;
    cudaError_t e = cudaEventSynchronize(ev[ne - 1]);
    if (e != cudaSuccess) return check_cuda(e, "cudaEventSynchronize");
    for (int k = 0; k + 1 < ne; ++k)
        if ((e = cudaEventElapsedTime(&ms[k], ev[k], ev[k + 1])) != cudaSuccess)
            return check_cuda(e, "cudaEventElapsedTime");
    return B200GSR_OK;
}

static int check_groups(int32_t num_groups, const b200gsr_group* groups, int32_t M) {
    if (num_groups < 0 || num_groups > B200GSR_MAX_GROUPS) return fail(B200GSR_ERR_UNSUPPORTED, "num_groups %d not in 0..%d", num_groups, B200GSR_MAX_GROUPS);
    if (num_groups > 0 && !groups) return fail(B200GSR_ERR_BAD_ARG, "groups is null");
    if (M < 1 || M > 16) return fail(B200GSR_ERR_BAD_ARG, "M=%d not in 1..16", M);
    long long total = 0;
    for (int g = 0; g < num_groups; ++g) {
        const b200gsr_group& gr = groups[g];
        if (gr.n < 0) return fail(B200GSR_ERR_BAD_ARG, "group %d: negative size", g);
        if (gr.n > 0 && (!gr.xyz || !gr.opacity || !gr.scaling || !gr.rotation || !gr.f_dc || (M > 1 && !gr.f_rest)))
            return fail(B200GSR_ERR_BAD_ARG, "group %d: null parameter pointer", g);
        if (gr.n > 0 && (reinterpret_cast<uintptr_t>(gr.rotation) & 15u))
            return fail(B200GSR_ERR_BAD_ARG, "group %d: rotation must be 16-byte aligned", g);
        total += gr.n;
    }
    if (total > 0x7fffffffLL) return fail(B200GSR_ERR_UNSUPPORTED, "more than 2^31-1 Gaussians");
    return B200GSR_OK;
}

int b200gsr_assemble_forward(int32_t num_groups, const b200gsr_group* groups, int32_t M, int32_t num_views, float shs_noise,
                             float scale_noise, const float* z_shs, const float* z_scales, uint64_t seed,
                             float* means3D, float* opacities, float* scales, float* rotations, float* shs,
                             void* stream) {
    int rc = check_groups(num_groups, groups, M);
    if (rc) return rc;
    if (!means3D || !opacities || !scales || !rotations || !shs) return fail(B200GSR_ERR_BAD_ARG, "null output pointer");
    if (num_views < 1 || num_views > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_BAD_ARG, "num_views %d not in 1..%d", num_views, B200GSR_MAX_VIEWS);
    GSR_RANGE_PUSH("b200gsr.assemble_fwd");
    rc = check_cuda(gsr_launch_assemble(false, num_groups, groups, nullptr, M, num_views, shs_noise, scale_noise, z_shs, z_scales,
                                        seed, means3D, opacities, scales, rotations, shs,
                                        static_cast<cudaStream_t>(stream)), "assemble_forward");
    GSR_RANGE_POP();
    return rc;
}

int b200gsr_assemble_backward(int32_t num_groups, const b200gsr_group* groups, const b200gsr_group_grad* grads,
                              int32_t M, int32_t num_views, float shs_noise, float scale_noise, const float* z_shs,
                              const float* z_scales, uint64_t seed, const float* d_means3D,
                              const float* d_opacities, const float* d_scales, const float* d_rotations,
                              const float* d_shs, void* stream) {
    int rc = check_groups(num_groups, groups, M);
    if (rc) return rc;
    if (num_groups > 0 && !grads) return fail(B200GSR_ERR_BAD_ARG, "grads is null");
    for (int g = 0; g < num_groups; ++g)
        if (groups[g].n > 0 && (!grads[g].xyz || !grads[g].opacity || !grads[g].scaling || !grads[g].rotation ||
                                !grads[g].f_dc || (M > 1 && !grads[g].f_rest)))
            return fail(B200GSR_ERR_BAD_ARG, "group %d: null gradient pointer", g);
    if (!d_means3D || !d_opacities || !d_scales || !d_rotations || !d_shs) return fail(B200GSR_ERR_BAD_ARG, "null gradient input");
    if (num_views < 1 || num_views > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_BAD_ARG, "num_views %d not in 1..%d", num_views, B200GSR_MAX_VIEWS);
    GSR_RANGE_PUSH("b200gsr.assemble_bwd");
    rc = check_cuda(gsr_launch_assemble(true, num_groups, groups, grads, M, num_views, shs_noise, scale_noise, z_shs, z_scales, seed,
                                        const_cast<float*>(d_means3D), const_cast<float*>(d_opacities),
                                        const_cast<float*>(d_scales), const_cast<float*>(d_rotations),
                                        const_cast<float*>(d_shs), static_cast<cudaStream_t>(stream)), "assemble_backward");
    GSR_RANGE_POP();
    return rc;
}

int b200gsr_disparity_forward(int32_t B, int32_t N, const float* depth_alpha, const float* focal, float* out_disp,
                              void* stats, void* stream) {
    if (B < 0 || N < 0 || ((B > 0 && N > 0) && (!depth_alpha || !focal || !out_disp || !stats)))
        return fail(B200GSR_ERR_BAD_ARG, "bad disparity_forward arguments");
    DeviceState* ds = device_state();
    if (!ds) return fail(B200GSR_ERR_CUDA, "cannot query the current CUDA device");
    return check_cuda(gsr_launch_disparity_fwd(B, N, depth_alpha, focal, out_disp, stats, ds->num_sms,
                                               static_cast<cudaStream_t>(stream)), "disparity_forward");
}

int b200gsr_disparity_backward_ex(int32_t B, int32_t N, const float* depth_alpha, const float* focal, const float* g_disp,
                                  const float* g_alpha, void* stats, float* d_depth_alpha, uint32_t flags, void* stream) {
    if (B < 0 || N < 0 || ((B > 0 && N > 0) && (!depth_alpha || !focal || !g_disp || !stats || !d_depth_alpha)))
        return fail(B200GSR_ERR_BAD_ARG, "bad disparity_backward arguments");
    DeviceState* ds = device_state();
    if (!ds) return fail(B200GSR_ERR_CUDA, "cannot query the current CUDA device");
    return check_cuda(gsr_launch_disparity_bwd(B, N, depth_alpha, focal, g_disp, g_alpha, stats, d_depth_alpha,
                                               (flags & B200GSR_BWD_DETERMINISTIC) != 0, ds->num_sms,
                                               static_cast<cudaStream_t>(stream)), "disparity_backward");
}

int b200gsr_disparity_backward(int32_t B, int32_t N, const float* depth_alpha, const float* focal, const float* g_disp,
                               const float* g_alpha, void* stats, float* d_depth_alpha, void* stream) {
    return b200gsr_disparity_backward_ex(B, N, depth_alpha, focal, g_disp, g_alpha, stats, d_depth_alpha, 0u, stream);
}

int b200gsr_frames(int32_t B, int32_t H, int32_t W, const float* color, const float* depth_alpha, const float* focal,
                   uint8_t* rgb8, uint8_t* depth8, void* stats, void* stream) {
    if (B < 1 || B > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_BAD_ARG, "frames: B = %d not in 1..%d", B, B200GSR_MAX_VIEWS);
    if (H < 1 || W < 1) return fail(B200GSR_ERR_BAD_ARG, "frames: image size %d x %d must be positive", W, H);
    if (!color || !depth_alpha || !focal || !rgb8 || !depth8 || !stats)
        return fail(B200GSR_ERR_BAD_ARG, "frames: null pointer");
    if ((reinterpret_cast<uintptr_t>(rgb8) | reinterpret_cast<uintptr_t>(depth8)) & 3u)
        return fail(B200GSR_ERR_BAD_ARG, "frames: rgb8 and depth8 must be 4-byte aligned");
    // the forwards' composite addresses a single view with its own height (unpadded), B > 1 views stacked
    const long long Hs = B == 1 ? H : (long long)B * gsr_grid(H, W).gy * GSR_TILE;
    if ((long long)B * H * W * 3 >= (1ll << 31) || Hs * W * 3 >= (1ll << 31))
        return fail(B200GSR_ERR_BAD_ARG, "frames: %d views of %d x %d are too large", B, W, H);
    DeviceState* ds = device_state();
    if (!ds) return fail(B200GSR_ERR_CUDA, "cannot query the current CUDA device");
    return check_cuda(gsr_launch_frames(B, H, W, (int)Hs, color, depth_alpha, focal, rgb8, depth8, stats, ds->num_sms,
                                        static_cast<cudaStream_t>(stream)), "frames");
}

#define GSR_ST(x) static_cast<cudaStream_t>(x)
int b200gsr_densify_stats(int32_t P, const float* viewspace_grad, const int32_t* radii, float* accum, float* denom,
                          float* max_radii2D, void* stream) {
    if (P < 0 || (P > 0 && (!viewspace_grad || !radii || !accum || !denom))) return fail(B200GSR_ERR_BAD_ARG, "bad densify_stats arguments");
    return check_cuda(gsr_densify_stats(P, viewspace_grad, radii, accum, denom, max_radii2D, GSR_ST(stream)), "densify_stats");
}
size_t b200gsr_densify_scratch_bytes(int32_t P) { return gsr_densify_scratch_bytes(P); }
int b200gsr_densify_plan(int32_t P, const float* accum, const float* denom, const float* scaling, const float* opacity,
                         float max_grad, float dense_extent, float min_opacity, float big_ws, float child_div,
                         void* scratch, uint32_t* totals5, void* stream) {
    if (P < 0 || !totals5 || (P > 0 && (!accum || !denom || !scaling || !opacity || !scratch)) || P > 0x0fffffff)
        return fail(B200GSR_ERR_BAD_ARG, "bad densify_plan arguments");
    return check_cuda(gsr_densify_plan(P, accum, denom, scaling, opacity, max_grad, dense_extent, min_opacity, big_ws,
                                       child_div, scratch, totals5, GSR_ST(stream)), "densify_plan");
}
int b200gsr_densify_map(int32_t P, int32_t N, const void* scratch, const uint32_t* totals5, int32_t* src_map,
                        int32_t* child_draw, void* stream) {
    if (P < 0 || N < 1 || (P > 0 && (!scratch || !totals5 || !src_map || !child_draw)))
        return fail(B200GSR_ERR_BAD_ARG, "bad densify_map arguments");
    return check_cuda(gsr_densify_map(P, N, scratch, totals5, src_map, child_draw, GSR_ST(stream)), "densify_map");
}
int b200gsr_compact_plan(int32_t P, const uint8_t* keep, void* scratch, int32_t* src_map, uint32_t* count, void* stream) {
    if (P < 0 || !count || (P > 0 && (!keep || !scratch || !src_map))) return fail(B200GSR_ERR_BAD_ARG, "bad compact_plan arguments");
    return check_cuda(gsr_compact_plan(P, keep, scratch, src_map, count, GSR_ST(stream)), "compact_plan");
}
int b200gsr_gather_rows(int32_t n_out, int32_t row_floats, const int32_t* src_map, const float* in, float* out,
                        int32_t zero_appended, void* stream) {
    if (n_out < 0 || row_floats < 0 || (n_out > 0 && row_floats > 0 && (!src_map || !in || !out)))
        return fail(B200GSR_ERR_BAD_ARG, "bad gather_rows arguments");
    return check_cuda(gsr_gather_rows(n_out, row_floats, src_map, in, out, zero_appended, GSR_ST(stream)), "gather_rows");
}
int b200gsr_split_children(int32_t n_out, int32_t first_child, float child_div, const int32_t* src_map,
                           const int32_t* child_draw, const float* xyz, const float* scaling, const float* rotation,
                           const float* z, float* xyz_out, float* scaling_out, void* stream) {
    if (n_out < 0 || first_child < 0 || (n_out > first_child && (!src_map || !child_draw || !xyz || !scaling || !rotation || !z || !xyz_out || !scaling_out)))
        return fail(B200GSR_ERR_BAD_ARG, "bad split_children arguments");
    return check_cuda(gsr_split_children(n_out, first_child, child_div, src_map, child_draw, xyz, scaling, rotation, z,
                                         xyz_out, scaling_out, GSR_ST(stream)), "split_children");
}
int b200gsr_kth_smallest(int32_t n, const float* v, uint32_t k, void* scratch, float* out, void* stream) {
    if (n < 0 || (n > 0 && (!v || !scratch || !out || k >= (uint32_t)n))) return fail(B200GSR_ERR_BAD_ARG, "bad kth_smallest arguments");
    DeviceState* ds = device_state();
    if (!ds) return fail(B200GSR_ERR_CUDA, "cannot query the current CUDA device");
    return check_cuda(gsr_kth_smallest(n, v, k, scratch, out, ds->num_sms, GSR_ST(stream)), "kth_smallest");
}

static int check_adam(int32_t n_tensors, const b200gsr_adam_tensor* tensors) {
    if (n_tensors < 0 || (n_tensors > 0 && !tensors)) return fail(B200GSR_ERR_BAD_ARG, "bad adam_step arguments");
    if (n_tensors > B200GSR_ADAM_MAX_TENSORS)
        return fail(B200GSR_ERR_UNSUPPORTED, "adam_step: %d tensors, at most %d per call", n_tensors, B200GSR_ADAM_MAX_TENSORS);
    for (int i = 0; i < n_tensors; ++i) {
        const b200gsr_adam_tensor& t = tensors[i];
        if (t.n < 0) return fail(B200GSR_ERR_BAD_ARG, "adam_step: tensor %d has a negative length", i);
        if (t.n > 0 && (!t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq))
            return fail(B200GSR_ERR_BAD_ARG, "adam_step: tensor %d has a null pointer", i);
    }
    return B200GSR_OK;
}

int b200gsr_adam_step(int32_t n_tensors, const b200gsr_adam_tensor* tensors, void* stream) {
    int rc = check_adam(n_tensors, tensors);
    if (rc) return rc;
    return check_cuda(gsr_launch_adam(n_tensors, tensors, GSR_ST(stream)), "adam_step");
}

int b200gsr_adam_step_dyn(int32_t n_tensors, const b200gsr_adam_tensor* tensors, const float* scalars, void* stream) {
    int rc = check_adam(n_tensors, tensors);
    if (rc) return rc;
    if (n_tensors > 0 && !scalars) return fail(B200GSR_ERR_BAD_ARG, "adam_step_dyn: scalars must be a device array [n, 6]");
    return check_cuda(gsr_launch_adam_dyn(n_tensors, tensors, scalars, GSR_ST(stream)), "adam_step_dyn");
}

int b200gsr_adam_step_dyn_live(int32_t n_tensors, const b200gsr_adam_tensor* tensors, const float* scalars,
                               const b200gsr_adam_live* live, void* stream) {
    int rc = check_adam(n_tensors, tensors);
    if (rc) return rc;
    if (n_tensors > 0 && !scalars) return fail(B200GSR_ERR_BAD_ARG, "adam_step_dyn_live: scalars must be a device array [n, 6]");
    if (n_tensors > 0 && !live) return fail(B200GSR_ERR_BAD_ARG, "adam_step_dyn_live: live must be a host array of n records");
    for (int i = 0; i < n_tensors; ++i)
        if (live[i].rows && (live[i].row_floats < 1 || tensors[i].n % live[i].row_floats))
            return fail(B200GSR_ERR_BAD_ARG, "adam_step_dyn_live: tensor %d: row_floats %d must be >= 1 and divide its "
                        "length %lld", i, live[i].row_floats, (long long)tensors[i].n);
    return check_cuda(gsr_launch_adam_dyn_live(n_tensors, tensors, scalars, live, GSR_ST(stream)), "adam_step_dyn_live");
}

int b200gsr_pair_report(const void* saved, uint32_t* report, void* stream) {
    if (!saved || !report) return fail(B200GSR_ERR_BAD_ARG, "pair_report: saved and report must be device pointers");
    return check_cuda(gsr_launch_pair_report(static_cast<const uint32_t*>(saved), report, GSR_ST(stream)), "pair_report");
}

size_t b200gsr_recon_l2_scratch_bytes(int32_t B, int32_t N) {
    return B < 1 || N < 1 ? 0 : (size_t)B * (size_t)gsr_l2_blocks(N) * sizeof(double);
}

int b200gsr_recon_l2(int32_t B, int32_t N, const float* image, const void* target, int32_t target_is_half,
                     int32_t n_targets, const int32_t* target_index, float weight, const void* grad_out,
                     void* loss_out, float* d_image, void* scratch, size_t scratch_bytes, void* stream) {
    if (B < 1 || N < 1 || n_targets < 1) return fail(B200GSR_ERR_BAD_ARG, "recon_l2: B %d, N %d and n_targets %d must be >= 1", B, N, n_targets);
    if (B > 65535) return fail(B200GSR_ERR_UNSUPPORTED, "recon_l2: at most 65535 views, got %d", B);
    if (target_is_half != 0 && target_is_half != 1) return fail(B200GSR_ERR_BAD_ARG, "recon_l2: target_is_half must be 0 or 1");
    if (!image || !target) return fail(B200GSR_ERR_BAD_ARG, "recon_l2: image and target must be device pointers");
    if (!loss_out && !d_image) return fail(B200GSR_ERR_BAD_ARG, "recon_l2: nothing to compute (loss_out and d_image are null)");
    if (d_image && !grad_out) return fail(B200GSR_ERR_BAD_ARG, "recon_l2: d_image needs grad_out");
    if (!target_index && B > n_targets)
        return fail(B200GSR_ERR_BAD_ARG, "recon_l2: without target_index view v uses target v, but B %d > n_targets %d", B, n_targets);
    if (loss_out && (!scratch || scratch_bytes < b200gsr_recon_l2_scratch_bytes(B, N) || (uintptr_t)scratch % 8))
        return fail(B200GSR_ERR_WORKSPACE, "recon_l2: scratch must be 8-byte aligned and hold %zu bytes (got %zu)",
                    b200gsr_recon_l2_scratch_bytes(B, N), scratch ? scratch_bytes : (size_t)0);
    GsrL2Args a;
    a.B = B; a.N = N; a.n_targets = n_targets;
    a.weight = weight;
    a.inv_n = 1.0f / (float)N;
    a.image = image; a.target = target; a.target_index = target_index; a.grad_out = grad_out;
    a.loss_out = loss_out; a.d_image = d_image; a.partials = static_cast<double*>(scratch);
    return check_cuda(gsr_launch_recon_l2(a, target_is_half != 0, GSR_ST(stream)), "recon_l2");
}

size_t b200gsr_tv_loss_scratch_bytes(int32_t B, int32_t C, int32_t H, int32_t W) {
    if (B < 1 || C < 1 || H < 2 || W < 2 || (long long)B * C * H * W > INT32_MAX) return 0;
    return (size_t)gsr_tv_blocks((long long)B * C, H, W, 1) * 2 * sizeof(double);      // the scalar path's grid
}

int b200gsr_tv_loss(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const float* grad_out, float* loss_out,
                    float* d_x, int32_t accumulate, void* scratch, size_t scratch_bytes, void* stream) {
    if (B < 1 || C < 1) return fail(B200GSR_ERR_BAD_ARG, "tv_loss: B %d and C %d must be >= 1", B, C);
    if (H < 2 || W < 2) return fail(B200GSR_ERR_BAD_ARG, "tv_loss: H %d and W %d must be >= 2", H, W);
    if ((long long)B * C * H * W > INT32_MAX)
        return fail(B200GSR_ERR_UNSUPPORTED, "tv_loss: at most 2^31 - 1 elements, got %lld", (long long)B * C * H * W);
    if (accumulate != 0 && accumulate != 1) return fail(B200GSR_ERR_BAD_ARG, "tv_loss: accumulate must be 0 or 1");
    if (!x) return fail(B200GSR_ERR_BAD_ARG, "tv_loss: x must be a device pointer");
    if (!loss_out && !d_x) return fail(B200GSR_ERR_BAD_ARG, "tv_loss: nothing to compute (loss_out and d_x are null)");
    if (d_x && !grad_out) return fail(B200GSR_ERR_BAD_ARG, "tv_loss: d_x needs grad_out");
    if (loss_out && (!scratch || scratch_bytes < b200gsr_tv_loss_scratch_bytes(B, C, H, W) || (uintptr_t)scratch % 8))
        return fail(B200GSR_ERR_WORKSPACE, "tv_loss: scratch must be 8-byte aligned and hold %zu bytes (got %zu)",
                    b200gsr_tv_loss_scratch_bytes(B, C, H, W), scratch ? scratch_bytes : (size_t)0);
    GsrTvArgs a;
    a.B = B; a.planes = B * C; a.H = H; a.W = W;
    const long long ch = (long long)C * (H - 1) * W, cw = (long long)C * H * (W - 1);
    a.inv_b = 1.0f / (float)B;              // torch's div by a CPU scalar: fp32(1 / fp32(n))
    a.inv_h = 1.0f / (float)ch;
    a.inv_w = 1.0f / (float)cw;
    a.count_h = (double)ch; a.count_w = (double)cw;
    a.x = x; a.grad_out = grad_out; a.loss_out = loss_out; a.d_x = d_x; a.accumulate = accumulate;
    a.partials = static_cast<double*>(scratch);
    return check_cuda(gsr_launch_tv_loss(a, GSR_ST(stream)), "tv_loss");
}

size_t b200gsr_scale_loss_scratch_bytes(int32_t rows) {
    return rows < 1 || 3LL * rows > INT32_MAX ? 0 : (size_t)gsr_l2_blocks(3 * rows) * sizeof(double);
}

int b200gsr_scale_loss(int32_t rows, const float* scales, const float* grad_out, float* loss_out, float* d_scales,
                       int32_t accumulate, void* scratch, size_t scratch_bytes, void* stream) {
    if (rows < 1) return fail(B200GSR_ERR_BAD_ARG, "scale_loss: rows %d must be >= 1", rows);
    if (3LL * rows > INT32_MAX) return fail(B200GSR_ERR_UNSUPPORTED, "scale_loss: at most 2^31 - 1 elements, got %lld", 3LL * rows);
    if (accumulate != 0 && accumulate != 1) return fail(B200GSR_ERR_BAD_ARG, "scale_loss: accumulate must be 0 or 1");
    if (!scales) return fail(B200GSR_ERR_BAD_ARG, "scale_loss: scales must be a device pointer");
    if (!loss_out && !d_scales) return fail(B200GSR_ERR_BAD_ARG, "scale_loss: nothing to compute (loss_out and d_scales are null)");
    if (d_scales && !grad_out) return fail(B200GSR_ERR_BAD_ARG, "scale_loss: d_scales needs grad_out");
    if (loss_out && (!scratch || scratch_bytes < b200gsr_scale_loss_scratch_bytes(rows) || (uintptr_t)scratch % 8))
        return fail(B200GSR_ERR_WORKSPACE, "scale_loss: scratch must be 8-byte aligned and hold %zu bytes (got %zu)",
                    b200gsr_scale_loss_scratch_bytes(rows), scratch ? scratch_bytes : (size_t)0);
    GsrScaleArgs a;
    a.rows = rows;
    a.inv_rows = 1.0f / (float)rows;        // MeanBackward0 / MeanBackward1: div by a CPU scalar
    a.inv_3 = 1.0f / 3.0f;
    a.scales = scales; a.grad_out = grad_out; a.loss_out = loss_out; a.d_scales = d_scales; a.accumulate = accumulate;
    a.partials = static_cast<double*>(scratch);
    return check_cuda(gsr_launch_scale_loss(a, GSR_ST(stream)), "scale_loss");
}

int b200gsr_scale_loss_live(int32_t B, int32_t num_groups, const b200gsr_group* groups, const int32_t* live,
                            const float* scales, const float* grad_out, float* loss_out, float* d_scales,
                            int32_t accumulate, void* scratch, size_t scratch_bytes, void* stream) {
    if (B < 1 || B > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: B %d not in 1..%d", B, B200GSR_MAX_VIEWS);
    if (num_groups < 1 || num_groups > B200GSR_MAX_GROUPS || !groups)
        return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: need a host array of 1..%d groups", B200GSR_MAX_GROUPS);
    if (!live) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: live must be a device array [num_groups]");
    GsrScaleLiveArgs a;
    long long P = 0;
    for (int g = 0; g < num_groups; ++g) {
        if (groups[g].n < 0) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: group %d has a negative n", g);
        a.start[g] = (int32_t)P;
        P += groups[g].n;
        if (P > INT32_MAX) return fail(B200GSR_ERR_UNSUPPORTED, "scale_loss_live: more than 2^31 - 1 rows");
    }
    if ((long long)B * P > INT32_MAX) return fail(B200GSR_ERR_UNSUPPORTED, "scale_loss_live: B * P too large");
    const int32_t rows = (int32_t)(B * P);
    if (rows < 1) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: the groups hold no row");
    if (3LL * rows > INT32_MAX) return fail(B200GSR_ERR_UNSUPPORTED, "scale_loss_live: at most 2^31 - 1 elements, got %lld", 3LL * rows);
    if (accumulate != 0 && accumulate != 1) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: accumulate must be 0 or 1");
    if (!scales) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: scales must be a device pointer");
    if (!loss_out && !d_scales) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: nothing to compute (loss_out and d_scales are null)");
    if (d_scales && !grad_out) return fail(B200GSR_ERR_BAD_ARG, "scale_loss_live: d_scales needs grad_out");
    if (loss_out && (!scratch || scratch_bytes < b200gsr_scale_loss_scratch_bytes(rows) || (uintptr_t)scratch % 8))
        return fail(B200GSR_ERR_WORKSPACE, "scale_loss_live: scratch must be 8-byte aligned and hold %zu bytes (got %zu)",
                    b200gsr_scale_loss_scratch_bytes(rows), scratch ? scratch_bytes : (size_t)0);
    a.start[num_groups] = (int32_t)P;
    a.rows = rows;
    a.inv_rows = 0.0f;                      // formed on the device from the live counts
    a.inv_3 = 1.0f / 3.0f;
    a.scales = scales; a.grad_out = grad_out; a.loss_out = loss_out; a.d_scales = d_scales; a.accumulate = accumulate;
    a.partials = static_cast<double*>(scratch);
    a.B = B; a.P = (int32_t)P; a.num_groups = num_groups; a.live = live;
    return check_cuda(gsr_launch_scale_loss_live(a, GSR_ST(stream)), "scale_loss_live");
}

int b200gsr_debug_counters(unsigned long long* device_counters) {
    g_stats = device_counters;
    return B200GSR_OK;
}

size_t b200gsr_dist2_scratch_bytes(int32_t P) { return P < 0 ? 0 : gsr_knn_scratch_bytes(P, nullptr); }

int b200gsr_dist2_knn3(int32_t P, const float* points, float* out, void* scratch, size_t scratch_bytes,
                       void* stream) {
    if (P < 0 || (P > 0 && (!points || !out || !scratch)))
        return fail(B200GSR_ERR_BAD_ARG, "bad dist2_knn3 arguments");
    if (scratch_bytes < gsr_knn_scratch_bytes(P, nullptr))
        return fail(B200GSR_ERR_WORKSPACE, "dist2_knn3 scratch too small: %zu < %zu", scratch_bytes,
                    gsr_knn_scratch_bytes(P, nullptr));
    return check_cuda(gsr_launch_knn(P, points, out, static_cast<uint8_t*>(scratch), static_cast<cudaStream_t>(stream)),
                      "dist2_knn3");
}

int b200gsr_sh_grad_expand(int32_t P, int32_t M, int32_t sh_degree, int32_t num_views, const float* means3D,
                           const float* dcol, size_t view_stride, float* d_shs, void* stream) {
    if (P < 0 || M < 1 || num_views < 1 || num_views > 64 || sh_degree < 0 || sh_degree > 3 ||
        M < (sh_degree + 1) * (sh_degree + 1) || view_stride < 3 * (size_t)P + 3 || (P > 0 && (!means3D || !dcol || !d_shs)))
        return fail(B200GSR_ERR_BAD_ARG, "bad sh_grad_expand arguments");
    return check_cuda(gsr_launch_sh_grad_expand(P, M, sh_degree, num_views, means3D, dcol, view_stride, d_shs,
                                                static_cast<cudaStream_t>(stream)), "sh_grad_expand");
}

// ---------------------------------------------------------------------------------------------
// Scene renders (include/b200gsr_scene.h): the views of a training step rendered straight from the raw parameter
// groups.  The forward is run_forward's kScene pass; the backward is the multi-view backward with the raw-leaf
// mode of project_bwd, views in order.
// ---------------------------------------------------------------------------------------------
// `sc` carries either the host noise arrays or (the _dyn entry points, `dyn`) the device records and seed, whose
// values the kernels trust; the host's tanfovx / tanfovy / sh_degree are not checked then, since they are not read.
static int check_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                       const GsrScene& sc, bool dyn) {
    if (B < 1 || B > B200GSR_MAX_VIEWS) return fail(B200GSR_ERR_UNSUPPORTED, "number of views %d not in 1..%d", B, B200GSR_MAX_VIEWS);
    if (!prm) return fail(B200GSR_ERR_BAD_ARG, "null view array");
    if (dyn && (!sc.dyn_views || !sc.dyn_seed))
        return fail(B200GSR_ERR_BAD_ARG, "views / seed must be device pointers to B step records and the seed");
    if (sc.live_call && !sc.live) return fail(B200GSR_ERR_BAD_ARG, "live must be a device array [num_groups]");
    if (!dyn && (!sc.shs_noise || !sc.scale_noise))
        return fail(B200GSR_ERR_BAD_ARG, "shs_noise / scale_noise must be host arrays of B coefficients");
    int rc = check_groups(num_groups, groups, prm[0].M);
    if (rc) return rc;
    long long total = 0;
    for (int g = 0; g < num_groups; ++g) total += groups[g].n;
    for (int v = 0; v < B; ++v) {
        const b200gsr_params& p = prm[v];
        if ((rc = check_size(p, v))) return rc;
        if (!p.bg || !p.viewmatrix || !p.projmatrix || !p.campos)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: bg/viewmatrix/projmatrix/campos must be device pointers", v);
        if (p.P != total) return fail(B200GSR_ERR_BAD_ARG, "view %d: P = %d but the groups hold %lld rows", v, p.P, total);
        if (p.M != prm[0].M || p.image_height != prm[0].image_height || p.image_width != prm[0].image_width)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: M and image size must equal view 0's", v);
        if (p.score_flag) return fail(B200GSR_ERR_UNSUPPORTED, "view %d: score_flag is not supported by the scene render", v);
        if (p.bg != prm[0].bg + 3 * v)
            return fail(B200GSR_ERR_BAD_ARG, "view %d: backgrounds must be one contiguous device array [B,3] (prm[v].bg = prm[0].bg + 3 v)", v);
        if (dyn) continue;
        if (p.sh_degree < 0 || p.sh_degree > 3) return fail(B200GSR_ERR_UNSUPPORTED, "view %d: sh_degree %d not in 0..3", v, p.sh_degree);
        if (p.M < (p.sh_degree + 1) * (p.sh_degree + 1))
            return fail(B200GSR_ERR_BAD_ARG, "view %d: M=%d inconsistent with sh_degree=%d (need (deg+1)^2 <= M)", v, p.M, p.sh_degree);
    }
    if ((long long)B * total > 0x3fffffffLL) return fail(B200GSR_ERR_UNSUPPORTED, "B * P too large");
    return B200GSR_OK;
}

// b200gsr_forward_scene and b200gsr_forward_scene_dyn: `sc` as check_scene's, completed with the outputs here
static int forward_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                         GsrScene sc, bool dyn, float* out_scales, float* out_color, float* out_depth_alpha,
                         int32_t* radii, void* scratch, size_t scratch_bytes, void* saved, size_t saved_bytes,
                         uint64_t max_pairs, uint32_t flags, uint32_t* host_notify, uint32_t notify_seq, void* stream) {
    int rc = check_scene(B, prm, num_groups, groups, sc, dyn);
    if (rc) return rc;
    if (flags & ~(B200GSR_FWD_NO_BACKWARD | B200GSR_FWD_DETERMINISTIC)) return fail(B200GSR_ERR_BAD_ARG, "unknown flags 0x%x", flags);
    if (!out_color || !out_depth_alpha || (prm[0].P > 0 && !radii) || !scratch || !saved)
        return fail(B200GSR_ERR_BAD_ARG, "null output/workspace pointer");
    sc.num_groups = num_groups; sc.groups = groups; sc.out_scales = out_scales;
    return run_forward(Pass::kScene, B, prm, nullptr, out_color, out_depth_alpha, radii, nullptr, scratch, scratch_bytes,
                       saved, saved_bytes, max_pairs, flags, host_notify, notify_seq, stream, &sc);
}

int b200gsr_forward_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                          const float* shs_noise, const float* scale_noise, uint64_t seed, float* out_scales,
                          float* out_color, float* out_depth_alpha, int32_t* radii, void* scratch, size_t scratch_bytes,
                          void* saved, size_t saved_bytes, uint64_t max_pairs, uint32_t flags, uint32_t* host_notify,
                          uint32_t notify_seq, void* stream) {
    GsrScene sc{};
    sc.shs_noise = shs_noise; sc.scale_noise = scale_noise; sc.seed = seed;
    return forward_scene(B, prm, num_groups, groups, sc, false, out_scales, out_color, out_depth_alpha, radii, scratch,
                         scratch_bytes, saved, saved_bytes, max_pairs, flags, host_notify, notify_seq, stream);
}

int b200gsr_forward_scene_dyn(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                              const b200gsr_step_view* views, const uint64_t* seed, float* out_scales,
                              float* out_color, float* out_depth_alpha, int32_t* radii, void* scratch,
                              size_t scratch_bytes, void* saved, size_t saved_bytes, uint64_t max_pairs, uint32_t flags,
                              uint32_t* host_notify, uint32_t notify_seq, void* stream) {
    GsrScene sc{};
    sc.dyn_views = views; sc.dyn_seed = reinterpret_cast<const unsigned long long*>(seed);
    return forward_scene(B, prm, num_groups, groups, sc, true, out_scales, out_color, out_depth_alpha, radii, scratch,
                         scratch_bytes, saved, saved_bytes, max_pairs, flags, host_notify, notify_seq, stream);
}

// The statistics arguments of b200gsr_backward_scene[_dyn]_stats (include/b200gsr_stats.h), after check_scene and the
// frozen mask's check.  -> whether any group gathers.
static int check_stats(int32_t B, int32_t num_groups, uint32_t frozen, const b200gsr_group_stats* stats, bool dyn,
                       int32_t stats_view, const int32_t* dyn_stats_view, bool& any) {
    any = false;
    if (!dyn && (stats_view < -1 || stats_view >= B))
        return fail(B200GSR_ERR_BAD_ARG, "stats_view %d not in -1..%d", stats_view, B - 1);
    for (int g = 0; g < num_groups && stats; ++g) {
        const b200gsr_group_stats& st = stats[g];
        if ((st.xyz_gradient_accum == nullptr) != (st.denom == nullptr))
            return fail(B200GSR_ERR_BAD_ARG, "group %d: xyz_gradient_accum and denom must both be set or both be null", g);
        if (st.xyz_gradient_accum == nullptr && st.max_radii2D != nullptr)
            return fail(B200GSR_ERR_BAD_ARG, "group %d: max_radii2D without xyz_gradient_accum and denom", g);
        if (st.xyz_gradient_accum == nullptr) continue;
        if ((frozen >> g) & 1u)
            return fail(B200GSR_ERR_BAD_ARG, "group %d: statistics on a frozen group (its rows would count in denom with "
                        "a zero gradient)", g);
        any = true;
    }
    if (any && dyn && !dyn_stats_view)
        return fail(B200GSR_ERR_BAD_ARG, "stats_view must be a device pointer to an int32 when a group gathers statistics");
    return B200GSR_OK;
}

// b200gsr_backward_scene, b200gsr_backward_scene_dyn (frozen = 0), their _frozen variants (include/b200gsr_frozen.h)
// and their _stats variants (include/b200gsr_stats.h, `with_stats`: d_means2D may be null)
static int backward_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                          const b200gsr_group_grad* grads, GsrScene sc, bool dyn, const float* d_scales,
                          const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                          const float* dL_ddepth_alpha, void* saved, size_t saved_bytes, uint64_t max_pairs,
                          float* d_means2D, uint32_t flags, uint32_t frozen, void* stream, bool with_stats = false,
                          const b200gsr_group_stats* stats = nullptr, int32_t stats_view = -1,
                          const int32_t* dyn_stats_view = nullptr) {
    int rc = check_scene(B, prm, num_groups, groups, sc, dyn);
    if (rc) return rc;
    if (flags & ~B200GSR_BWD_DETERMINISTIC) return fail(B200GSR_ERR_BAD_ARG, "unknown flags 0x%x", flags);
    if (frozen >> num_groups)      // num_groups <= B200GSR_MAX_GROUPS < 32 (check_scene)
        return fail(B200GSR_ERR_BAD_ARG, "frozen mask 0x%x has bits at or above num_groups %d", frozen, num_groups);
    bool gathers = false;
    if (with_stats && (rc = check_stats(B, num_groups, frozen, stats, dyn, stats_view, dyn_stats_view, gathers)))
        return rc;
    if (num_groups > 0 && !grads) return fail(B200GSR_ERR_BAD_ARG, "grads is null");
    for (int g = 0; g < num_groups; ++g)
        if (groups[g].n > 0 && !((frozen >> g) & 1u) && (!grads[g].xyz || !grads[g].opacity || !grads[g].scaling || !grads[g].rotation ||
                                !grads[g].f_dc || (prm[0].M > 1 && !grads[g].f_rest)))
            return fail(B200GSR_ERR_BAD_ARG, "group %d: null gradient pointer", g);
    const int P = prm[0].P;
    if (P == 0) return B200GSR_OK;
    if (!radii || !out_depth_alpha || !dL_dcolor || !dL_ddepth_alpha || !saved || (!d_means2D && !with_stats))
        return fail(B200GSR_ERR_BAD_ARG, "null saved-state/gradient pointer");
    GsrBwdArgs a;
    if ((rc = setup_backward(true, B, prm, radii, out_depth_alpha, dL_dcolor, dL_ddepth_alpha, saved, saved_bytes,
                             max_pairs, (flags & B200GSR_BWD_DETERMINISTIC) != 0, stream, a)))
        return rc;
    sc.num_groups = num_groups; sc.groups = groups; sc.grads = grads; sc.d_scales = d_scales; sc.frozen = frozen;
    if (gathers) {
        sc.stats = stats;
        sc.stats_view = stats_view;
        sc.dyn_stats_view = dyn_stats_view;
    } else {
        sc.stats_view = -1;
    }
    a.scene = &sc;
    a.g_begin = 0; a.g_end = P;
    prof_mark_bwd(0, a.stream);
    GSR_RANGE_PUSH("b200gsr.scene.composite_bwd");
    rc = check_cuda(gsr_launch_composite_bwd(a), "composite_bwd");
    GSR_RANGE_POP();
    if (rc) return rc;
    prof_mark_bwd(1, a.stream);
    GSR_RANGE_PUSH("b200gsr.scene.project_bwd");
    for (int v = 0; v < B && !rc; ++v) {      // in view order: view 0 writes the leaf gradients, later views add
        a.prm = prm[v]; a.view = v;
        a.d_means2D = d_means2D ? d_means2D + 3 * (size_t)P * v : nullptr;
        // the STATS kernel where it has work: every view under _dyn (the view to gather is read on the device) or
        // without d_means2D; by value, only the launch of the view that gathers.  The other launches are _frozen's.
        sc.stats_mode = with_stats && (dyn || !d_means2D || (gathers && v == stats_view));
        rc = check_cuda(gsr_launch_project_bwd(a), "project_bwd");
    }
    GSR_RANGE_POP();
    if (rc) return rc;
    prof_mark_bwd(2, a.stream);
    if (g_prof.max_calls > 0 && g_prof.nbwd < g_prof.max_calls) ++g_prof.nbwd;
    return B200GSR_OK;
}

int b200gsr_backward_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                           const b200gsr_group_grad* grads, const float* shs_noise, const float* scale_noise,
                           uint64_t seed, const float* d_scales, const int32_t* radii, const float* out_depth_alpha,
                           const float* dL_dcolor, const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                           uint64_t max_pairs, float* d_means2D, uint32_t flags, void* stream) {
    GsrScene sc{};
    sc.shs_noise = shs_noise; sc.scale_noise = scale_noise; sc.seed = seed;
    return backward_scene(B, prm, num_groups, groups, grads, sc, false, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, 0u, stream);
}

int b200gsr_backward_scene_dyn(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                               const b200gsr_group_grad* grads, const b200gsr_step_view* views, const uint64_t* seed,
                               const float* d_scales, const int32_t* radii, const float* out_depth_alpha,
                               const float* dL_dcolor, const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                               uint64_t max_pairs, float* d_means2D, uint32_t flags, void* stream) {
    GsrScene sc{};
    sc.dyn_views = views; sc.dyn_seed = reinterpret_cast<const unsigned long long*>(seed);
    return backward_scene(B, prm, num_groups, groups, grads, sc, true, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, 0u, stream);
}

int b200gsr_backward_scene_frozen(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                                  const b200gsr_group_grad* grads, const float* shs_noise, const float* scale_noise,
                                  uint64_t seed, const float* d_scales, const int32_t* radii,
                                  const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha,
                                  void* saved, size_t saved_bytes, uint64_t max_pairs, float* d_means2D,
                                  uint32_t flags, uint32_t frozen_groups, void* stream) {
    GsrScene sc{};
    sc.shs_noise = shs_noise; sc.scale_noise = scale_noise; sc.seed = seed;
    return backward_scene(B, prm, num_groups, groups, grads, sc, false, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, frozen_groups, stream);
}

int b200gsr_backward_scene_dyn_frozen(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                      const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                      const b200gsr_step_view* views, const uint64_t* seed, const float* d_scales,
                                      const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                      const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                                      uint64_t max_pairs, float* d_means2D, uint32_t flags, uint32_t frozen_groups,
                                      void* stream) {
    GsrScene sc{};
    sc.dyn_views = views; sc.dyn_seed = reinterpret_cast<const unsigned long long*>(seed);
    return backward_scene(B, prm, num_groups, groups, grads, sc, true, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, frozen_groups, stream);
}

int b200gsr_backward_scene_stats(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                                 const b200gsr_group_grad* grads, const float* shs_noise, const float* scale_noise,
                                 uint64_t seed, const float* d_scales, const int32_t* radii,
                                 const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha,
                                 void* saved, size_t saved_bytes, uint64_t max_pairs, float* d_means2D,
                                 uint32_t flags, uint32_t frozen_groups, const b200gsr_group_stats* stats,
                                 int32_t stats_view, void* stream) {
    GsrScene sc{};
    sc.shs_noise = shs_noise; sc.scale_noise = scale_noise; sc.seed = seed;
    return backward_scene(B, prm, num_groups, groups, grads, sc, false, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, frozen_groups, stream,
                          true, stats, stats_view, nullptr);
}

int b200gsr_backward_scene_dyn_stats(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                     const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                     const b200gsr_step_view* views, const uint64_t* seed, const float* d_scales,
                                     const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                     const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                                     uint64_t max_pairs, float* d_means2D, uint32_t flags, uint32_t frozen_groups,
                                     const b200gsr_group_stats* stats, const int32_t* stats_view, void* stream) {
    GsrScene sc{};
    sc.dyn_views = views; sc.dyn_seed = reinterpret_cast<const unsigned long long*>(seed);
    return backward_scene(B, prm, num_groups, groups, grads, sc, true, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, frozen_groups, stream,
                          true, stats, -1, stats_view);
}

int b200gsr_forward_scene_dyn_live(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                   const b200gsr_group* groups, const b200gsr_step_view* views, const uint64_t* seed,
                                   float* out_scales, float* out_color, float* out_depth_alpha, int32_t* radii,
                                   void* scratch, size_t scratch_bytes, void* saved, size_t saved_bytes,
                                   uint64_t max_pairs, uint32_t flags, uint32_t* host_notify, uint32_t notify_seq,
                                   const int32_t* live, void* stream) {
    GsrScene sc{};
    sc.dyn_views = views; sc.dyn_seed = reinterpret_cast<const unsigned long long*>(seed);
    sc.live = live; sc.live_call = true;
    return forward_scene(B, prm, num_groups, groups, sc, true, out_scales, out_color, out_depth_alpha, radii, scratch,
                         scratch_bytes, saved, saved_bytes, max_pairs, flags, host_notify, notify_seq, stream);
}

int b200gsr_backward_scene_dyn_live(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                    const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                    const b200gsr_step_view* views, const uint64_t* seed, const float* d_scales,
                                    const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                    const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                                    uint64_t max_pairs, float* d_means2D, uint32_t flags, uint32_t frozen_groups,
                                    const b200gsr_group_stats* stats, const int32_t* stats_view,
                                    const int32_t* live, void* stream) {
    GsrScene sc{};
    sc.dyn_views = views; sc.dyn_seed = reinterpret_cast<const unsigned long long*>(seed);
    sc.live = live; sc.live_call = true;
    return backward_scene(B, prm, num_groups, groups, grads, sc, true, d_scales, radii, out_depth_alpha, dL_dcolor,
                          dL_ddepth_alpha, saved, saved_bytes, max_pairs, d_means2D, flags, frozen_groups, stream,
                          true, stats, -1, stats_view);
}

int b200gsr_mark_visible(int32_t P, const float* means3D, const float* viewmatrix,
                         const float* projmatrix, uint8_t* visible, void* stream) {
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !visible)))
        return fail(B200GSR_ERR_BAD_ARG, "bad mark_visible arguments");
    return check_cuda(gsr_launch_mark_visible(P, means3D, viewmatrix, projmatrix, visible,
                                              static_cast<cudaStream_t>(stream)), "mark_visible");
}

}  // extern "C"
