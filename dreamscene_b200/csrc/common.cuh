// Shared device-side definitions for the H100 (sm_90a) Gaussian rasterizer kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>

#include "../../include/b200gsr_reserve.h"

#define GSR_TILE 16
#define GSR_NEAR_Z 0.2f
#define GSR_ALPHA_MIN (1.0f / 255.0f)
#define GSR_ALPHA_MAX 0.99f
#define GSR_T_STOP 1e-4f
#define GSR_LOG2E 1.4426950408889634f
#define GSR_LN2 0.6931471805599453f

// One (tile, Gaussian) pair as consumed by the composite kernels; also the per-Gaussian
// "geom" record written by project_sh (the sort epilogue copies geom[idx] -> sorted[pos]).
// 48 bytes = 3 x 16 B, so 8 consecutive lanes reading one 16-B part each hit 8 distinct
// 4-bank groups (stride 12 words) -> conflict-free LDS.128, and a record moves as three
// 16-byte cp.async copies.
struct __align__(16) GsrRec {
    // part 0: everything the per-warp cull test needs
    float px, py;   // pixel-space mean
    uint32_t ext;   // half2 (ext_x, ext_y): conservative half extents of {alpha >= 1/255}
    float A;        // scaled conic: log2(G) = A*dx*dx + B*dx*dy + C*dy*dy  (GSR_EXACT_EXP: raw conic.x)
    // part 1
    float B, C;     //   A = -0.5*log2e*conic.x, B = -log2e*conic.y, C = -0.5*log2e*conic.z
    float opacity;
    float depth;    // view-space z
    // part 2
    float r, g, b;  // colour (SH evaluated, +0.5, clamped >= 0) or colors_precomp
    uint32_t idx;   // Gaussian index
};
static_assert(sizeof(GsrRec) == 48, "record must be 48 bytes");

struct GsrTileGrid {
    int gx, gy, ntiles;
};

__host__ __device__ inline GsrTileGrid gsr_grid(int H, int W) {
    GsrTileGrid g;
    g.gx = (W + GSR_TILE - 1) / GSR_TILE;
    g.gy = (H + GSR_TILE - 1) / GSR_TILE;
    g.ntiles = g.gx * g.gy;
    return g;
}

// header words in the saved buffer (uint32[GSR_H_WORDS])
enum { GSR_H_NUM_PAIRS = 0, GSR_H_MAX_PAIRS = 1, GSR_H_NUM_TILES = 2, GSR_H_OVERFLOW = 3,
       GSR_H_NUM_BIG = 4, GSR_H_NUM_NONEMPTY = 5,
       GSR_H_BWD_QUEUE = 8,       // [8, 8+GSR_NQUEUE): work-queue counters of composite_bwd; zeroed by the
                                  // forward's scan kernel and restored to zero by project_bwd, so a saved
                                  // buffer can be back-propagated any number of times without a memset
       GSR_H_BWD_QUEUE_DET = 16,  // [16, 16+GSR_NQUEUE): the same for the second deterministic backward pass; zeroed
                                  // by the deterministic forward, restored to zero by det_resolve_kernel
       GSR_H_BWD_FILL = 32,       // [32, 64): items per size class of the backward's work lists (written by the
                                  // forward's composite kernel, zeroed by its scan kernel)
       GSR_H_WORDS = 64 };
// Backward work items = (tile, 8x4-pixel block) pairs that blended at least one entry, binned by the
// forward into GSR_BWD_CLASSES size classes of the block's consumed list length (two classes per power
// of two); the backward pops the longest first.  List of class k: bwd_items[k * num_tiles * 8 ...].
#define GSR_BWD_CLASSES 32
__host__ __device__ inline int gsr_bwd_class(uint32_t n) {     // n >= 1
#ifdef __CUDA_ARCH__
    const int e = 31 - __clz((int)n);
#else
    int e = 0; while (e < 31 && (n >> (e + 1)) != 0u) ++e;
#endif
    const int k = 2 * e + (e > 0 ? (int)((n >> (e - 1)) & 1u) : 0);
    return k < GSR_BWD_CLASSES - 1 ? k : GSR_BWD_CLASSES - 1;
}
// counters in scratch
// The tile work queue is split into GSR_NQUEUE sub-queues (tile w lives in queue w % NQUEUE): one
// shared counter would serialise every fetch at the ~30 ns same-address L2 atomic rate.
#define GSR_NQUEUE 8
#define GSR_NCOUNTERS 128
enum { GSR_C_FWD_QUEUE = 0 };

#define GSR_SORT_SMALL_MAX 4096   // keys sorted by the 256-thread kernel (256 x 16 items)
#define GSR_SORT_BIG_CHUNK 16384  // keys per smem chunk of the 1024-thread kernel (1024 x 16 items)
// Tile counters/cursors are privatised into GSR_COPIES arrays (copy = (gaussian_idx>>5) & mask):
// same-address L2 atomics serialise at ~30 ns each, so the hottest tile bounds the kernel.
#define GSR_COPIES 16
// Block-multisplit binning (default when the tile grid fits in shared memory): a CTA of 1024
// threads owns GSR_MS_ITEMS*1024 consecutive Gaussians and histograms their tile hits in smem, so
// global atomics drop from one per (Gaussian, tile) pair to one per (CTA, touched tile).
#define GSR_MS_ITEMS 4
// Number of multisplit CTAs for P (virtual) Gaussians: at most 4096 Gaussians per CTA; a scene that
// would fill less than one wave (2 CTAs x 132 SMs on H100) is spread over the whole wave instead, down to 256
// Gaussians per CTA, so that every SM carries the same load.
#define GSR_MS_WAVE_CTAS 264
__host__ __device__ inline int gsr_ms_blocks(long long P) {
    const long long full = (P + 1024 * GSR_MS_ITEMS - 1) / (1024 * GSR_MS_ITEMS);
    if (full >= GSR_MS_WAVE_CTAS) return (int)full;
    const long long fine = (P + 255) / 256;
    return (int)(fine < 1 ? 1 : (fine < GSR_MS_WAVE_CTAS ? fine : GSR_MS_WAVE_CTAS));
}
#define GSR_MS_MAX_TILES 12288   // 4 B x tiles of dynamic smem (48 KB); 12 tiles per thread in the scan kernel
__host__ __device__ inline bool gsr_use_multisplit(int ntiles) { return ntiles <= GSR_MS_MAX_TILES; }
// uint32 words at the start of scratch that must be zero before the count kernel runs: the queue counters and the
// per-tile pair counters (on the multisplit path two arrays, the pair counts and the padded counts; all GSR_COPIES on
// the large-grid fallback).  The multisplit projection zeroes them in its prologue; otherwise the forward issues a
// memset.  Host code only.
inline size_t gsr_counter_words(const b200gsr_scratch_layout& sl, int ntiles) {
    return (gsr_use_multisplit(ntiles) ? sl.tile_count + 2 * (size_t)ntiles * sizeof(uint32_t) : sl.tile_cursor) / sizeof(uint32_t);
}
// Multisplit path: the key scatter writes every CTA's slice of a tile rounded up to whole 32-byte sectors (4 keys, the
// pad slots hold ~0ull) into a padded key buffer at the end of scratch, and the tile sort compacts each tile's padded
// segment into saved.keys.  A slice has at most 3 pad keys, so the buffer holds max_pairs + 3 * CTAs * tiles keys
// (capped so that a padded position fits in 32 bits).  P = virtual Gaussians.  Host code only.
inline uint32_t gsr_pad_key_capacity(uint64_t max_pairs, int P, int ntiles) {
    const uint64_t cap = max_pairs + 3ull * (uint64_t)gsr_ms_blocks(P) * (uint64_t)ntiles;
    return (uint32_t)(cap < 0xfffffff0ull ? cap : 0xfffffff0ull);
}
inline size_t gsr_pad_keys_offset(const b200gsr_scratch_layout& sl, int P, int ntiles) {
    return (sl.ms_hist + (size_t)gsr_ms_blocks(P) * ntiles * sizeof(uint32_t) + 255) / 256 * 256;
}

// ---- deterministic mode (B200GSR_FWD_DETERMINISTIC / B200GSR_BWD_DETERMINISTIC) ------------------------
// Float atomics sum in whatever order the warps commit.  Deterministic mode commits integer images of the
// partials instead: integer addition is associative, so the sum no longer depends on that order.
//   gradients: per (Gaussian, component) the largest |partial| is found first (pass A, atomicMax of the float
//              bits); pass B adds round(partial * 2^s) with s = GSR_DET_FIX_BITS - exponent(largest) into int64.
//              A partial is then < 2^(K+1) in magnitude, and a Gaussian receives at most 8 commits per tile of
//              its view, so with at most GSR_DET_MAX_VIEW_TILES tiles (8192^2 pixels) a sum stays below
//              2^21 * 2^41 = 2^62: no overflow, with a factor 2 to spare.  Quantisation error <= 2^-(K+1) of the
//              component's largest partial per commit.
//   important score: every commit is a warp's summed blend weight; a Gaussian's score is at most its view's
//              pixel count (2^26), so a fixed scale 2^GSR_DET_SCORE_BITS keeps the sum below 2^62.
// The constants are fixed (never derived from the image or the view count): a sum depends only on the set
// of partials, so one view of a multi-view render reproduces the single-view result bit for bit.
#define GSR_DET_FIX_BITS 40
#define GSR_DET_MAX_VIEW_TILES (1 << 18)
#define GSR_DET_SCORE_BITS 36
#define GSR_DET_COMPONENTS 10     // per-Gaussian gradient accumulators used of the 12 in a dgeom row

// Offsets of the deterministic accumulators, appended to the saved buffer after bwd_items (0 = absent).
struct GsrDetLayout {
    size_t dmax;       // uint32[P][10]: float bits of the largest |partial| per (Gaussian, component)
    size_t dfx;        // int64[P][10]: fixed-point sums
    size_t score_fx;   // int64[P]: fixed-point important score
    size_t total;
};

__host__ __device__ inline double gsr_pow2(int s) {   // exact 2^s for -1022 <= s <= 1023
    const unsigned long long b = (unsigned long long)(s + 1023) << 52;
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)b);
#else
    double d;
    __builtin_memcpy(&d, &b, sizeof(d));
    return d;
#endif
}
// Scale exponent s for a component whose largest |partial| has the float bits `max_bits` (finite, sign clear).
__host__ __device__ inline int gsr_det_shift(uint32_t max_bits) {
    int e = (int)(max_bits >> 23);   // biased exponent
    if (e == 0) e = 1;               // zero or subnormal: bounded by the smallest normal binade
    return GSR_DET_FIX_BITS - (e - 127);
}
__host__ __device__ inline bool gsr_det_finite(uint32_t max_bits) { return max_bits < 0x7f800000u; }
__host__ __device__ inline long long gsr_det_quantise(float x, int shift) {
    return llrint((double)x * gsr_pow2(shift));
}
// The summed component; NaN when any partial was NaN or infinite (the float atomics give a non-finite sum too).
__host__ __device__ inline float gsr_det_dequantise(long long sum, uint32_t max_bits) {
    if (!gsr_det_finite(max_bits)) return nanf("");
    return (float)((double)sum * gsr_pow2(-gsr_det_shift(max_bits)));
}
__host__ __device__ inline long long gsr_det_score_quantise(float w) {
    return llrint((double)w * gsr_pow2(GSR_DET_SCORE_BITS));
}
__host__ __device__ inline float gsr_det_score_dequantise(long long sum) {
    return (float)((double)sum * gsr_pow2(-GSR_DET_SCORE_BITS));
}

#ifdef __CUDACC__
// ---- 128-bit global access helpers -------------------------------------------------------
__device__ __forceinline__ float4 ldg_f4(const void* p) {
    return *reinterpret_cast<const float4*>(p);
}
__device__ __forceinline__ void stg_na_f4(void* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// Default build: exp via ONE MUFU (ex2.approx on a conic pre-scaled by log2 e), T recovery in the
// backward via rcp.approx.  -DGSR_EXACT_EXP builds the parity-diagnostic variant
// (libb200gsr_exact.so): the record keeps the UNSCALED conic, the exponent is evaluated with
// individually rounded fp32 ops in the oracle's operation order (oracle/splat_ref.py::composite),
// exp is expf() and the reciprocal an IEEE division.  It exists to show that the forward outliers
// against the oracle are exp-approximation artefacts at the discontinuous 1/255 and 1e-4 tests
// (tools/parity_stats.py measures both builds) and what the approximation buys (ms).
#ifdef GSR_EXACT_EXP
#define GSR_PX_GRAD_SCALE 1.0f
__device__ __forceinline__ float rcp_approx(float x) { return __fdiv_rn(1.0f, x); }
#else
#define GSR_PX_GRAD_SCALE GSR_LN2
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif

// ---- densification statistics ------------------------------------------------------------
// |(gx, gy)|, the reference's torch.norm(grad[:, :2], dim=-1), as sqrt(fma(gx, gx, gy * gy)) with every step rounded
// to nearest: the contraction nvcc chose for sqrtf(gx * gx + gy * gy), now fixed.  densify_stats_kernel and
// project_bwd's STATS mode both call it, so the statistics gathered inside the backward equal those of
// b200gsr_densify_stats over the stored d_means2D rows bit for bit.  The product and the FMA are written in PTX
// because __fmul_rn / __fmaf_rn reorder densify_stats_kernel's two loads (same arithmetic, different SASS).
__device__ __forceinline__ float gsr_screen_grad_norm(float gx, float gy) {
    float s;
    asm("{\n\t.reg .f32 yy;\n\tmul.rn.f32 yy, %2, %2;\n\tfma.rn.f32 %0, %1, %1, yy;\n\t}" : "=f"(s) : "f"(gx), "f"(gy));
    return __fsqrt_rn(s);
}

// ---- shared-memory address helper (cp.async destinations) ----------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
#endif  // __CUDACC__

// ---- kernel launchers (defined in the .cu files, called from api.cu) ---------------------
// Scene renders (b200gsr_forward_scene / b200gsr_backward_scene): the projection reads each group's raw leaves and
// applies the activations and the view's augmentation itself instead of reading packed per-view arrays.
struct GsrScene {
    int num_groups;
    const b200gsr_group* groups;         // host array of num_groups records
    const b200gsr_group_grad* grads;     // host array (backward): leaf gradient destinations
    const float* shs_noise;              // host [B]: per-view SH noise coefficient (0 = off)
    const float* scale_noise;            // host [B]: per-view scale noise coefficient (0 = off)
    unsigned long long seed;
    float* out_scales;                   // forward: [B,P,3] augmented scales, or null
    const float* d_scales;               // backward: [B,P,3] incoming gradient of those scales, or null
    // b200gsr_*_scene_dyn: device [B] per-view records and the device seed, read by the kernels in place of
    // shs_noise / scale_noise / seed and the views' tanfovx / tanfovy / sh_degree (both null otherwise)
    const b200gsr_step_view* dyn_views;
    const unsigned long long* dyn_seed;
    // backward (b200gsr_backward_scene[_dyn]_frozen): bit g = group g is frozen; its leaves get no gradient and
    // composite_bwd / project_bwd run their FROZEN instantiations.  0 = the default kernels.
    uint32_t frozen;    // backward (b200gsr_backward_scene[_dyn]_stats): project_bwd runs its STATS instantiation, which takes a null
    // d_means2D and gathers the densification statistics of `stats` (host array [num_groups], or null) in the launch
    // of the view stats_view (by value) or *dyn_stats_view (the _dyn entry point).  false = the other kernels.
    bool stats_mode;
    const b200gsr_group_stats* stats;
    int32_t stats_view;
    const int32_t* dyn_stats_view;
    // b200gsr_*_scene_dyn_live: device [num_groups] live row counts (include/b200gsr_reserve.h); project_sh /
    // project_bwd run their LIVE instantiations.  Null otherwise.
    const int32_t* live;
    bool live_call;                      // a _live entry point: `live` must be set
};

struct GsrFwdArgs {
    b200gsr_params prm;
    const float *means3D, *shs, *colors, *opac, *scales, *rots, *cov3d;
    float *out_color, *out_depth_alpha, *score;
    int32_t* radii;
    uint8_t *scratch, *saved;
    b200gsr_scratch_layout sl;
    b200gsr_saved_layout vl;
    uint32_t max_pairs;
    uint32_t* host_notify;
    uint32_t notify_seq;
    uint32_t flags;        // B200GSR_FWD_*
    bool det;              // B200GSR_FWD_DETERMINISTIC: `dl` locates the fixed-point accumulators in `saved`
    GsrDetLayout dl;
    // multi-view (b200gsr_forward_views): the views are stacked vertically into one image of
    // num_views * gy_view tile rows; view v's Gaussians are the virtual Gaussians [v*P_view, (v+1)*P_view).
    // Single-view calls: view = 0, num_views = 1, P_view = prm.P, gy_view = tile rows of the image.
    int view, num_views, P_view, gy_view;
    int num_sms;           // of the current device (cached per device in api.cu)
    unsigned long long* stats;
    cudaStream_t stream;
    const GsrScene* scene; // scene render: the raw leaves replace means3D .. cov3d (null otherwise)
};

struct GsrBwdArgs {
    b200gsr_params prm;
    const float *means3D, *shs, *colors, *opac, *scales, *rots, *cov3d;
    const int32_t* radii;
    const float *out_depth_alpha, *dL_dcolor, *dL_ddepth_alpha;
    uint8_t* saved;     // counters + gradient accumulators inside are consumed and restored
    b200gsr_saved_layout vl;
    uint32_t max_pairs;
    float *d_means3D, *d_means2D, *d_shs, *d_colors, *d_opac, *d_scales, *d_rots, *d_cov3d;
    int view, num_views, P_view, gy_view;   // see GsrFwdArgs
    int accumulate;        // project_bwd adds into the gradient outputs instead of overwriting (views sharing a parameter)
    int g_begin, g_end;    // Gaussian range of the project_bwd stage (chunked launches)
    int dsh_coefs;         // coefficients per row of d_shs (0 = M, the reference layout)
    bool det;              // B200GSR_BWD_DETERMINISTIC: fixed-point accumulation, see GsrDetLayout
    GsrDetLayout dl;
    int num_sms;
    unsigned long long* stats;   // optional device counters (b200gsr_debug_counters); selects the STATS kernels
    cudaStream_t stream;
    const GsrScene* scene;       // scene render: leaf gradients of the raw parameters (null otherwise)
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device) instead of on every
// launch: `done` is a per-call-site bit mask indexed by device ordinal.
template <typename F>
inline cudaError_t gsr_smem_once(F func, int bytes, std::atomic<unsigned long long>& done) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const unsigned long long bit = 1ull << (dev & 63);
    if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
    return e;
}

// geo: the score pass's geometry-only projection (no SH row or colour read, no backward state)
cudaError_t gsr_launch_project(const GsrFwdArgs& a, bool geo);
cudaError_t gsr_launch_count(const GsrFwdArgs& a);         // multisplit path: per-tile pair counts
cudaError_t gsr_launch_scan(const GsrFwdArgs& a);          // exclusive scan + work order + host notify
cudaError_t gsr_launch_scatter(const GsrFwdArgs& a);       // append keys to tile lists
cudaError_t gsr_launch_sort(const GsrFwdArgs& a, cudaStream_t side, cudaEvent_t fork, cudaEvent_t join);   // per-tile sort (2 kernels, concurrent when `side` is given)
cudaError_t gsr_launch_composite_fwd(const GsrFwdArgs& a);
cudaError_t gsr_launch_composite_bwd(const GsrBwdArgs& a);
// score pass (b200gsr_score_views): score-only compositing into score_acc (float [P_view], or int64 [P_view] with
// a.det); score_finish converts an int64 accumulator to float
cudaError_t gsr_launch_composite_score(const GsrFwdArgs& a, void* score_acc);
cudaError_t gsr_launch_score_finish(int n, const unsigned long long* score_fx, float* score, cudaStream_t s);
cudaError_t gsr_launch_project_bwd(const GsrBwdArgs& a);
cudaError_t gsr_launch_sh_grad_expand(int P, int M, int deg, int nviews, const float* means3D, const float* dcol,
                                      size_t stride, float* d_shs, cudaStream_t s);
cudaError_t gsr_launch_mark_visible(int P, const float* means3D, const float* view,
                                    const float* proj, uint8_t* visible, cudaStream_t s);

// scene assembly (assemble.cu)
cudaError_t gsr_launch_assemble(bool backward, int num_groups, const b200gsr_group* groups,
                                const b200gsr_group_grad* grads, int M, int B, float c_shs, float c_scale,
                                const float* z_shs, const float* z_scales, unsigned long long seed,
                                float* means3D, float* opac, float* scales, float* rots, float* shs, cudaStream_t s);

// disparity post-processing (postprocess.cu)
cudaError_t gsr_launch_disparity_fwd(int B, int N, const float* da, const float* focal, float* out, void* stats,
                                     int num_sms, cudaStream_t s);
cudaError_t gsr_launch_disparity_bwd(int B, int N, const float* da, const float* focal, const float* g_out,
                                     const float* g_alpha, void* stats, float* d_da, bool deterministic, int num_sms,
                                     cudaStream_t s);
// 8-bit video frames of B stacked views (postprocess.cu; b200gsr_frames)
cudaError_t gsr_launch_frames(int B, int H, int W, int Hs, const float* color, const float* da, const float* focal,
                              uint8_t* rgb8, uint8_t* depth8, void* stats, int num_sms, cudaStream_t s);

// densification / pruning (densify.cu)
cudaError_t gsr_densify_stats(int P, const float* vs_grad, const int32_t* radii, float* accum, float* denom,
                              float* max_radii, cudaStream_t s);
size_t gsr_densify_scratch_bytes(int P);
cudaError_t gsr_densify_plan(int P, const float* accum, const float* denom, const float* scaling, const float* opacity,
                             float max_grad, float dense_extent, float min_opacity, float big_ws, float child_div, void* scratch,
                             uint32_t* totals5, cudaStream_t s);
cudaError_t gsr_densify_map(int P, int N, const void* scratch, const uint32_t* totals5, int32_t* src_map,
                            int32_t* child_draw, cudaStream_t s);
cudaError_t gsr_compact_plan(int P, const uint8_t* keep, void* scratch, int32_t* src_map, uint32_t* count, cudaStream_t s);
cudaError_t gsr_gather_rows(int n_out, int row_floats, const int32_t* src_map, const float* in, float* out,
                            int zero_appended, cudaStream_t s);
cudaError_t gsr_split_children(int n_out, int first_child, float child_div, const int32_t* src_map, const int32_t* child_draw,
                               const float* xyz, const float* scaling, const float* rotation, const float* z,
                               float* xyz_out, float* scaling_out, cudaStream_t s);
cudaError_t gsr_kth_smallest(int n, const float* v, uint32_t k, void* scratch, float* out, int num_sms, cudaStream_t s);

// simple_knn replacement (knn.cu)
size_t gsr_knn_scratch_bytes(int P, int* max_cells_out);
cudaError_t gsr_launch_knn(int P, const float* pts, float* out, uint8_t* scratch, cudaStream_t s);

// ---- Adam step (optim.cu) ----------------------------------------------------------------------
// One launch over the virtual concatenation of up to B200GSR_ADAM_MAX_TENSORS tensors: every CTA owns
// GSR_ADAM_CHUNK consecutive elements of one tensor and finds it from the table, which travels in the kernel
// parameters (32 x 80 B).  A chunk is a multiple of 4 elements, so in a tensor whose four arrays are 16-byte
// aligned every chunk starts aligned; only the tensor's last chunk can have a scalar tail.
#define GSR_ADAM_THREADS 256
#define GSR_ADAM_VEC 4                                               // float4 per thread
#define GSR_ADAM_CHUNK (GSR_ADAM_THREADS * GSR_ADAM_VEC * 4)         // 4096 elements per CTA
struct GsrAdamEntry {
    float* p;
    const float* g;
    float* m;
    float* v;
    long long n;
    long long block0;      // first CTA of this tensor
    float w, beta2, omb2, eps, step_size, bc2_sqrt;
    int vec;               // all four pointers 16-byte aligned
};
struct GsrAdamTable {
    GsrAdamEntry e[B200GSR_ADAM_MAX_TENSORS];
    int count;
};

// Fills `tab` from n <= B200GSR_ADAM_MAX_TENSORS records (empty tensors dropped) -> number of CTAs.
inline long long gsr_adam_plan(int n, const b200gsr_adam_tensor* t, GsrAdamTable* tab) {
    long long blocks = 0;
    int k = 0;
    for (int i = 0; i < n; ++i) {
        if (t[i].n <= 0) continue;
        GsrAdamEntry& e = tab->e[k++];
        e.p = t[i].param; e.g = t[i].grad; e.m = t[i].exp_avg; e.v = t[i].exp_avg_sq;
        e.n = t[i].n;
        e.block0 = blocks;
        e.w = t[i].lerp_weight; e.beta2 = t[i].beta2; e.omb2 = t[i].one_minus_beta2; e.eps = t[i].eps;
        e.step_size = t[i].step_size; e.bc2_sqrt = t[i].bc2_sqrt;
        const uintptr_t any = reinterpret_cast<uintptr_t>(e.p) | reinterpret_cast<uintptr_t>(e.g) |
                              reinterpret_cast<uintptr_t>(e.m) | reinterpret_cast<uintptr_t>(e.v);
        e.vec = (any & 15u) == 0;
        blocks += (e.n + GSR_ADAM_CHUNK - 1) / GSR_ADAM_CHUNK;
    }
    tab->count = k;
    return blocks;
}
// The entry CTA b works on (b < the plan's CTA count).
__host__ __device__ inline int gsr_adam_find(const GsrAdamTable& tab, long long b) {
    int t = 0;
#pragma unroll
    for (int k = 1; k < B200GSR_ADAM_MAX_TENSORS; ++k)
        if (k < tab.count && b >= tab.e[k].block0) t = k;
    return t;
}
// Elements [start, end) of CTA b within its entry; [start, vend) is a whole number of float4s (empty unless e.vec),
// [vend, end) the scalar rest.
struct GsrAdamChunk { long long start, vend, end; };
__host__ __device__ inline GsrAdamChunk gsr_adam_chunk(const GsrAdamEntry& e, long long b) {
    GsrAdamChunk c;
    c.start = (b - e.block0) * GSR_ADAM_CHUNK;
    c.end = c.start + GSR_ADAM_CHUNK < e.n ? c.start + GSR_ADAM_CHUNK : e.n;
    c.vend = e.vec ? c.start + ((c.end - c.start) & ~3LL) : c.start;
    return c;
}
cudaError_t gsr_launch_adam(int n, const b200gsr_adam_tensor* t, cudaStream_t s);
// b200gsr_adam_step_dyn: the scalars of record i are read from scalars[6 i ..] in device memory
cudaError_t gsr_launch_adam_dyn(int n, const b200gsr_adam_tensor* t, const float* scalars, cudaStream_t s);
// b200gsr_adam_step_dyn_live: as _dyn, each tensor cut to its live elements (*live[i].rows * live[i].row_floats)
cudaError_t gsr_launch_adam_dyn_live(int n, const b200gsr_adam_tensor* t, const float* scalars,
                                     const b200gsr_adam_live* live, cudaStream_t s);
// b200gsr_pair_report: fold a forward's pair count and overflow flag (its saved header) into report[2]
cudaError_t gsr_launch_pair_report(const uint32_t* header, uint32_t* report, cudaStream_t s);

// ---- b200gsr_recon_l2 (include/b200gsr_loss.h, csrc/loss.cu) ------------------------------------------------------
// One CTA per GSR_L2_CHUNK elements of one view (16 per thread); with a loss, each CTA writes one double partial to
// scratch[v * gsr_l2_blocks(N) + b] and a second launch sums a view's partials in a fixed order.
constexpr int GSR_L2_THREADS = 256;
constexpr int GSR_L2_CHUNK = GSR_L2_THREADS * 16;
inline long long gsr_l2_blocks(int32_t N) { return ((long long)N + GSR_L2_CHUNK - 1) / GSR_L2_CHUNK; }
struct GsrL2Args {
    int32_t B, N, n_targets;
    float weight, inv_n;           // inv_n = fp32(1 / fp32(N)), the reciprocal torch's mean backward multiplies by
    const float* image;
    const void* target;
    const int32_t* target_index;   // NULL: view v uses target v
    const void* grad_out;          // with d_image
    void* loss_out;                // NULL: no loss
    float* d_image;                // NULL: no gradient
    double* partials;              // with loss_out
};
cudaError_t gsr_launch_recon_l2(const GsrL2Args& a, bool half_target, cudaStream_t s);

// ---- b200gsr_tv_loss / b200gsr_scale_loss (include/b200gsr_loss.h, csrc/loss.cu) ------------------------------------
// Total variation: a warp task is GSR_TV_ROWS rows x 32 lanes x V columns of one plane (V = 4 on the float4 path, 1 on
// the scalar one), GSR_L2_THREADS / 32 tasks per CTA; with a loss each CTA writes one (h, w) pair of double partials.
constexpr int GSR_TV_ROWS = 8;
inline long long gsr_tv_blocks(long long planes, int32_t H, int32_t W, int V) {
    const long long tasks = planes * ((H + GSR_TV_ROWS - 1) / GSR_TV_ROWS) * ((W + 32LL * V - 1) / (32LL * V));
    return (tasks + GSR_L2_THREADS / 32 - 1) / (GSR_L2_THREADS / 32);
}
struct GsrTvArgs {
    int32_t B, planes, H, W;        // planes = B C
    float inv_b, inv_h, inv_w;      // fp32(1 / B), fp32(1 / (C (H-1) W)), fp32(1 / (C H (W-1))): torch's reciprocals
    double count_h, count_w;        // C (H-1) W, C H (W-1)
    const float* x;
    const float* grad_out;          // with d_x
    float* loss_out;                // NULL: no loss
    float* d_x;                     // NULL: no gradient
    int32_t accumulate;
    double* partials;               // with loss_out: 2 per CTA of the scalar path's grid (the larger one)
};
cudaError_t gsr_launch_tv_loss(const GsrTvArgs& a, cudaStream_t s);
// Scale loss over n = 3 rows elements: CTA b owns elements [b GSR_L2_CHUNK, (b + 1) GSR_L2_CHUNK) as recon_l2 does.
struct GsrScaleArgs {
    int32_t rows;
    float inv_rows, inv_3;          // fp32(1 / rows), fp32(1 / 3)
    const float* scales;
    const float* grad_out;
    float* loss_out;
    float* d_scales;
    int32_t accumulate;
    double* partials;               // with loss_out: gsr_l2_blocks(3 rows)
};
cudaError_t gsr_launch_scale_loss(const GsrScaleArgs& a, cudaStream_t s);
// b200gsr_scale_loss_live: rows = B P over the groups' capacities; element e of view row r is live iff r's row in its
// group is below live[group].  inv_rows is formed on the device from B sum(live).
struct GsrScaleLiveArgs : GsrScaleArgs {
    int32_t B, P, num_groups;
    int32_t start[B200GSR_MAX_GROUPS + 1];   // first row of group g in a view; start[num_groups] = P
    const int32_t* live;
};
cudaError_t gsr_launch_scale_loss_live(const GsrScaleLiveArgs& a, cudaStream_t s);
