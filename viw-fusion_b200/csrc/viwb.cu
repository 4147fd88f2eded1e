// viwb.cu -- host side of libviwb.so: the C ABI of include/viwb.h over the CUDA kernels in this directory.
//
// Lowers viwb_problem tables to the device layout of layout.cuh (sorting visual factors by landmark, building the
// per-frame-pair gather lists, compacting the active tangent columns), runs the fixed launch sequence of one
// Estimator::optimization() (estimator.cpp:1383-1896) for a whole batch of windows and brings results back.
// There is no host arithmetic on the data path and no CPU fallback: without a CUDA device every entry point fails.
//
// The same file compiles with -DVIWB_HOST_EMU (g++, no CUDA) into the test-only kernel-logic emulation used by
// the `not gpu` tests (tests/emu); that build is never part of libviwb.so.
#include "../../include/viwb.h"
#include "kernels_marg.cuh"
#include "kernels_fused.cuh"
#include "kernels_lk.cuh"
#include "kernels_preint.cuh"
#include "kernels_feat.cuh"
#include "kernels_init.cuh"
#include "kernels_detect.cuh"
#include "kernels_track.cuh"
#include "kernels_fm.cuh"

#include <algorithm>
#include <map>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

using namespace viwb;

// ====================================================================================== device abstraction
#ifdef VIWB_HOST_EMU
typedef void *stream_t;
// poison fresh 'device' memory with NaN bytes so that reads of never-written data show up in the CPU tests
static int dev_malloc(void **p, size_t n) { *p = malloc(n ? n : 1); if (*p) memset(*p, 0xFF, n ? n : 1); return *p ? 0 : 1; }
static void dev_free(void *p) { free(p); }
static int dev_h2d(void *d, const void *h, size_t n, stream_t) { if (n) memcpy(d, h, n); return 0; }
static int dev_d2h(void *h, const void *d, size_t n, stream_t) { if (n) memcpy(h, d, n); return 0; }
static int dev_d2d(void *d, const void *s, size_t n, stream_t) { if (n) memcpy(d, s, n); return 0; }
static int dev_sync(stream_t) { return 0; }
static int host_alloc(void **p, size_t n) { *p = malloc(n ? n : 1); return *p ? 0 : 1; }
static void host_free(void *p) { free(p); }
static const char *dev_errstr(int) { return "emulation"; }
#define VIWB_EMU_NT 1
template <typename F>
static void emu_launch(F f, const BatchDev &bd, int gx, int gy, size_t smem_bytes, int mode) {
#ifdef VIWB_EMU_STRICT
    std::vector<double> sm((smem_bytes + 7) / 8);       // sanitizer build: exactly the dynamic shared memory the launch asks for
#else
    std::vector<double> sm(smem_bytes / 8 + 64);
#endif
    for (int by = 0; by < gy; by++) for (int bx = 0; bx < gx; bx++) f(bd, bx, by, 0, 1, sm.data(), mode);
}
#define NT(n) 1
enum { PRE_WPB = 1 };      // warps per block of the pre-integration kernels (kernels_preint.cuh): one per emulated block
#else
#include <cuda_runtime.h>
typedef cudaStream_t stream_t;
static int dev_malloc(void **p, size_t n) { return (int)cudaMalloc(p, n ? n : 1); }
static void dev_free(void *p) { cudaFree(p); }
static int dev_h2d(void *d, const void *h, size_t n, stream_t s) { return n ? (int)cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s) : 0; }
static int dev_d2h(void *h, const void *d, size_t n, stream_t s) { return n ? (int)cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, s) : 0; }
static int dev_d2d(void *d, const void *s_, size_t n, stream_t s) { return n ? (int)cudaMemcpyAsync(d, s_, n, cudaMemcpyDeviceToDevice, s) : 0; }
static int dev_sync(stream_t s) { return (int)cudaStreamSynchronize(s); }
static int host_alloc(void **p, size_t n) { return (int)cudaHostAlloc(p, n ? n : 1, cudaHostAllocDefault); }
static void host_free(void *p) { cudaFreeHost(p); }
static const char *dev_errstr(int e) { return cudaGetErrorString((cudaError_t)e); }
// optional per-kernel CUDA-event profiler (bench.py's live roofline timing); off by default
struct Profiler {
    bool on = false;
    std::vector<std::string> names; std::vector<double> ms; std::vector<long long> count;
    struct Rec { int idx; cudaEvent_t a, b; };
    std::vector<Rec> pending;
    int index(const char *n) { for (size_t i = 0; i < names.size(); i++) if (names[i] == n) return (int)i; names.push_back(n); ms.push_back(0); count.push_back(0); return (int)names.size() - 1; }
    void begin(const char *n, cudaStream_t s) { if (!on) return; Rec r; r.idx = index(n); cudaEventCreate(&r.a); cudaEventCreate(&r.b); cudaEventRecord(r.a, s); pending.push_back(r); }
    void end(cudaStream_t s) { if (!on) return; cudaEventRecord(pending.back().b, s); }
    void collect() { for (auto &r : pending) { cudaEventSynchronize(r.b); float t = 0; cudaEventElapsedTime(&t, r.a, r.b); ms[r.idx] += t; count[r.idx]++; cudaEventDestroy(r.a); cudaEventDestroy(r.b); } pending.clear(); }
};
static Profiler g_prof;
#define DEF_KERNEL2(name, maxnt, minb) \
    __global__ void __launch_bounds__(maxnt, minb) name##_kernel(BatchDev bd, int mode) { \
        extern __shared__ double viwb_smem[]; \
        name##_block(bd, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, viwb_smem, mode); }
#define DEF_KERNEL(name, maxnt) DEF_KERNEL2(name, maxnt, 1)
#ifndef LIN_VIS_MINB
#define LIN_VIS_MINB 3
#endif
DEF_KERNEL(vis_expand, 128)
DEF_KERNEL(setup, 128)
DEF_KERNEL(prior_setup, 256)
DEF_KERNEL2(lin_vis, 128, LIN_VIS_MINB)
DEF_KERNEL(lm_reduce, 128)
#ifndef LSM_MINB
#define LSM_MINB 4      // 128 registers, 4 blocks / SM: the spills of the IMU evaluation (10 threads of the block) cost less than the idle SM (r02n: 0.38 -> 0.25 ms per launch)
#endif
DEF_KERNEL2(lin_small, 128, LSM_MINB)
DEF_KERNEL(asm_items, 128)
// SOLVE_NT (kernels_solve.cuh): 256 threads and a C2 window's shared memory fit three windows per SM.  solve_wide runs the same block function
// with 384 threads, two per SM, for batches whose widest window leaves no room for a third block (solve_threads); -DSOLVE_NT=384 builds both at 384.
DEF_KERNEL2(solve, SOLVE_NT, SOLVE_NT <= 256 ? 3 : 2)
enum { SOLVE_WIDE_NT = 384 };
VIWB_D void solve_wide_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) { solve_block(bd, bx, by, tid, nt, smem, mode); }
DEF_KERNEL2(solve_wide, SOLVE_WIDE_NT, 2)
#ifndef LVL_MINB
#define LVL_MINB 4
#endif
DEF_KERNEL2(lin_vis_lm, LMB_FACTORS, LVL_MINB)
DEF_KERNEL2(lin_vis_lm_wide, LMB_FACTORS, 3)
DEF_KERNEL(asm_pairs_wide, 128)
#ifndef PAIR_RED_NT
#define PAIR_RED_NT 256
#endif
DEF_KERNEL(pair_reduce, PAIR_RED_NT)
DEF_KERNEL2(syrk_mma, SYRK_NT, 4)
DEF_KERNEL(reanchor, 32)
DEF_KERNEL2(marg_prep, 256, 2)
DEF_KERNEL2(marg_eig, 256, 3)
#ifndef MARG_TRI_NT
#define MARG_TRI_NT 256
#endif
DEF_KERNEL2(marg_tri, MARG_TRI_NT, 3)
DEF_KERNEL(marg_ql, 32)
DEF_KERNEL2(marg_apply, 128, 4)
DEF_KERNEL(outlier, 128)
#define NT(n) (n)
#endif
// Every kernel launch goes through KERNEL.  An empty grid launches nothing.  Otherwise the library issues kernel<<<(gx, gy), nt, smem>>>args on the
// context's stream inside the profiler's bracket, and the emulation build runs the statements of the variadic tail instead (block functions called
// block by block, one host thread per block: the grids of the emulation are sized with NT(n) = 1).  Either way ctx->launches counts exactly the
// launches issued, so viwb_launch_count equals the sum of the profile's launches.
#ifdef VIWB_HOST_EMU
#define KERNEL(ctx, pname, gx, gy, nt, smem, kernel, args, ...) do { if ((gx) > 0 && (gy) > 0) { __VA_ARGS__; (ctx)->launches++; } } while (0)
#else
#define KERNEL(ctx, pname, gx, gy, nt, smem, kernel, args, ...) \
    do { if ((gx) > 0 && (gy) > 0) { g_prof.begin(pname, (ctx)->stream); kernel<<<dim3((gx), (gy)), (nt), (smem), (ctx)->stream>>> args; g_prof.end((ctx)->stream); (ctx)->launches++; } } while (0)
#endif
// the BatchDev kernels (DEF_KERNEL): name##_kernel in the library, name##_block in the emulation; profiled as name, or name_marg in mode 1
#define LAUNCH(ctx, name, bd, gx, gy, nt, smem_bytes, mode) \
    KERNEL(ctx, (mode) == 1 ? #name "_marg" : #name, gx, gy, nt, smem_bytes, name##_kernel, (bd, mode), emu_launch(name##_block, bd, gx, gy, smem_bytes, mode))

// one device slab + one pinned host staging slab; cached in the context so that the host-buffer entry points do not
// pay cudaMalloc / cudaHostAlloc on every call
struct Arena { char *dev = nullptr; size_t dev_cap = 0; char *host = nullptr; size_t host_cap = 0; bool busy = false; };
static void arena_release(Arena &a) { if (a.dev) dev_free(a.dev); if (a.host) host_free(a.host); a = Arena(); }
static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static bool g_timing = getenv("VIWB_TIMING") != nullptr;
static bool g_marg_one_kernel = getenv("VIWB_MARG_ONE_KERNEL") != nullptr;      // measurement aid: tred2 + tql2 in one block-per-window kernel (marg_eig)
struct viwb_context {
    int device;
    stream_t stream;        // the stream all work of this context is issued on (own_stream unless viwb_set_stream gave another)
    stream_t own_stream;    // created by viwb_create, destroyed by viwb_destroy; a caller's stream is never destroyed here
    long long launches;
    long long h2d_bytes;    // bytes of window tables uploaded so far (the wire format, not the caller's tables)
    std::string err;
    bool attrs_set;
    Arena arena;
    struct viwb_lk_batch *lk1;      // one-stream LK state behind viwb_lk_track / viwb_track_checked
    struct viwb_detector *det1;     // one-stream detector behind viwb_set_mask / viwb_good_features_to_track
};

static int fail(viwb_context *ctx, int code, const std::string &msg) { if (ctx) ctx->err = msg; return code; }
// CUDA's current device is per host thread: every entry point binds the context's device before touching it, so that
// contexts can be driven from any thread (one context per thread at a time)
static inline void bind_device(const viwb_context *ctx) {
#ifndef VIWB_HOST_EMU
    if (ctx) { int cur = -1; if (cudaGetDevice(&cur) != cudaSuccess || cur != ctx->device) cudaSetDevice(ctx->device); }   // the host application may have switched devices in between
#else
    (void)ctx;
#endif
}
#define CK(call) do { int e_ = (call); if (e_) return fail(ctx, VIWB_ERR_CUDA, std::string(#call) + ": " + dev_errstr(e_)); } while (0)
// the error of a launch that failed at issue time (a bad configuration, no kernel image for the device); every entry point that launches asks once
static int launch_status(viwb_context *ctx) {
#ifndef VIWB_HOST_EMU
    const int e = (int)cudaGetLastError();
    if (e) return fail(ctx, VIWB_ERR_CUDA, std::string("kernel launch: ") + dev_errstr(e));
#endif
    (void)ctx;
    return VIWB_OK;
}
// the kernels' dynamic shared memory above the default limit; cudaFuncSetAttribute applies to the current device, so once per context
static int ensure_attrs(viwb_context *ctx) {
#ifndef VIWB_HOST_EMU
    if (!ctx->attrs_set) {
        CK(cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(solve_smem_doubles(SOLVE_NT, TFIX * (TFIX + 1) / 2, TFIX) * 8)));
        CK(cudaFuncSetAttribute(solve_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(solve_smem_doubles(SOLVE_WIDE_NT, TFIX * (TFIX + 1) / 2, TFIX) * 8)));
        CK(cudaFuncSetAttribute(lin_vis_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(lin_vis_smem_doubles(128) * 8)));
        CK(cudaFuncSetAttribute(lin_vis_lm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(lin_vis_run_smem_doubles() * 8)));
        CK(cudaFuncSetAttribute(lin_vis_lm_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(lin_vis_lm_smem_doubles(true) * 8)));
        CK(cudaFuncSetAttribute(syrk_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(syrk_mma_smem_doubles() * 8)));
        CK(cudaFuncSetAttribute(marg_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(marg_prep_smem_doubles(256, 100) * 8)));
        CK(cudaFuncSetAttribute(marg_tri_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(marg_eig_smem_doubles(256, 100) * 8)));
        CK(cudaFuncSetAttribute(marg_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(marg_apply_smem_doubles(128, 100) * 8)));
        CK(cudaFuncSetAttribute(marg_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(marg_eig_smem_doubles(256, 100) * 8)));
        CK(cudaFuncSetAttribute(det_corners_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)det_tile_smem_bytes()));
        CK(cudaFuncSetAttribute(det_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)det_select_smem_bytes()));
        ctx->attrs_set = true;
    }
#endif
    (void)ctx;
    return 0;
}

static size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

// One buffer of a one-shot entry point (staged): an input uploaded before the launch, an output downloaded after it, or device scratch.  `dev`
// is the kernel argument that receives the device address; an input or output without a host pointer is neither allocated nor copied (NULL).
struct Stage { void **dev; const void *in; void *out; size_t bytes; bool scratch; };
template <typename T> static Stage stage_in(T *&dev, const void *host, size_t bytes) { return {(void **)&dev, host, nullptr, bytes, false}; }
template <typename T> static Stage stage_out(T *&dev, void *host, size_t bytes) { return {(void **)&dev, nullptr, host, bytes, false}; }
template <typename T> static Stage stage_tmp(T *&dev, size_t bytes) { return {(void **)&dev, nullptr, nullptr, bytes, true}; }
// A one-shot entry point: one device block laid out align_up-aligned, the inputs up, launch() (KERNEL calls), the outputs down, then synchronise
// before the block is freed.  Copies run in the order of `bufs`.
template <typename Launch> static int staged(viwb_context *ctx, const char *what, std::initializer_list<Stage> bufs, Launch launch) {
    bind_device(ctx);
    size_t tot = 0;
    for (const Stage &b : bufs) if (b.scratch || b.in || b.out) tot += align_up(b.bytes);
    char *d = nullptr;
    int e = dev_malloc((void **)&d, tot), rc = VIWB_OK;
    if (e) return fail(ctx, VIWB_ERR_CUDA, std::string(what) + ": " + dev_errstr(e));
    size_t o = 0;
    for (const Stage &b : bufs) {
        const bool used = b.scratch || b.in || b.out;
        *b.dev = used ? d + o : nullptr;
        if (used) o += align_up(b.bytes);
        if (b.in && !e) e = dev_h2d(*b.dev, b.in, b.bytes, ctx->stream);
    }
    if (!e) { launch(); rc = launch_status(ctx); }
    for (const Stage &b : bufs) if (b.out && !e && !rc) e = dev_d2h(b.out, *b.dev, b.bytes, ctx->stream);
    const int es = dev_sync(ctx->stream);
    if (!e) e = es;
    dev_free(d);
    if (rc) return rc;
    return e ? fail(ctx, VIWB_ERR_CUDA, std::string(what) + ": " + dev_errstr(e)) : VIWB_OK;
}

#include "lk_host.inl"
#include "detect_host.inl"
#include "track_host.inl"
#include "features_host.inl"

// ====================================================================================== batch
struct HostPrior { int valid, n, nb; int block_id[NB], block_idx[NB]; std::vector<double> x0, J, r; };
struct viwb_batch {
    int B;
    BatchDev bd;
    Arena arena; bool arena_cached;      // cached: borrowed from the context (host-buffer calls), else owned
    size_t out_bytes, out_off;           // staging of the results inside the pinned slab: after the inputs (the upload is not waited for, so the regions must not overlap)
    std::vector<int> prior_n;            // n of the prior each window will produce (known from the plan)
    int prior_nmax;
    WinWork *work_init_dev;              // pristine solver states, copied to bd.work at the start of every run
    std::vector<WinMeta> meta;
    std::vector<int> out_mode;        // 0: prior computed on the device, 1: input prior passes through, 2: invalid / none
    std::vector<HostPrior> in_prior;
    std::vector<int> state_sizes;
    size_t total_state;
    double algorithmic_bytes;
    bool any_marg;
    int max_iter;
    double max_time;       // max_solver_time_in_seconds (0 = off): checked on the host between rounds, like Ceres' wall-clock test
    // viwb_features_batch_create: the lists it was built from and their generation then; x_fix [B][SFIX] the uploaded fixed states (the fill copies
    // them into x_init beside the landmarks), fm_off [2][B] each window's state_off and lm_off for the feedback kernels.  NULL / unused otherwise.
    const viwb_features *fs; long long fs_gen;
    double *x_fix; int *fm_off;
};

static void opts_from(const viwb_options *o, Opts &d) {
    d.max_num_iterations = o->max_num_iterations; d.max_invalid = o->max_num_consecutive_invalid_steps; d.jacobi_scaling = o->jacobi_scaling;
    d.function_tolerance = o->function_tolerance; d.gradient_tolerance = o->gradient_tolerance; d.parameter_tolerance = o->parameter_tolerance;
    d.initial_radius = o->initial_trust_region_radius; d.max_radius = o->max_trust_region_radius; d.min_radius = o->min_trust_region_radius;
    d.min_relative_decrease = o->min_relative_decrease; d.min_lm_diagonal = o->min_lm_diagonal; d.max_lm_diagonal = o->max_lm_diagonal;
}

extern "C" void viwb_default_options(viwb_options *o) {
    o->max_num_iterations = 8; o->max_solver_time_in_seconds = 0;
    o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
    o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32;
    o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32;
    o->max_num_consecutive_invalid_steps = 5; o->jacobi_scaling = 1;
}
extern "C" void viwb_default_globals(viwb_globals *g) {
    g->G[0] = 0; g->G[1] = 0; g->G[2] = 9.81007;
    g->vis_sqrt_info[0] = 460.0 / 1.5; g->vis_sqrt_info[1] = 0; g->vis_sqrt_info[2] = 0; g->vis_sqrt_info[3] = 460.0 / 1.5;
    g->plane_sqrt_info[0] = 100.0; g->plane_sqrt_info[1] = 100.0; g->plane_sqrt_info[2] = 20.0;
    g->huber_delta = 1.0;
}

static double window_algorithmic_bytes(const viwb_problem &p, int iters) {
    // SURVEY 8(d): B_solve = iters * B_iter + B_marg
    double R = 0, pg = p.num_landmarks;
    for (int b = 0; b < NB; b++) if (p.block_flags[b] & VIWB_BLOCK_PRESENT) { pg += blk_size(b); if (!(p.block_flags[b] & VIWB_BLOCK_CONSTANT)) R += blk_tsize(b); }
    const double n = (p.prior && p.prior->valid) ? p.prior->n : 0;
    const double b_iter = 112.0 * p.num_vis + 2296.0 * p.num_imu + 624.0 * p.num_wheel + 4.0 * p.num_plane + 8 * (n * n + 2 * n) + 8 * pg + 2 * 8 * (R * R + R) + 8 * pg;
    int nv0 = 0; std::vector<char> l0(p.num_landmarks > 0 ? p.num_landmarks : 1, 0);
    for (int i = 0; i < p.num_vis; i++) if (p.vis_frame_i[i] == 0) { nv0++; l0[p.vis_landmark[i]] = 1; }
    double m = 15; for (int k = 0; k < p.num_landmarks; k++) m += l0[k];
    const double nn = std::max(n, 76.0);
    const double b_marg = 112.0 * nv0 + 2296 + (p.num_wheel ? 624 : 0) + (p.num_plane ? 4 : 0) + 8 * (n * n + 2 * n) + 8 * ((m + nn) * (m + nn) + (m + nn)) + 8 * (nn * nn + nn);
    return iters * b_iter + b_marg;
}

static void batch_free(viwb_context *ctx, viwb_batch *b);

// ---- per-window lowering, phase 1: validation, sizes, active columns, and the plan (no offsets yet): the paths of the window's solver linearisation
// and marginalisation, and the sizes of those paths' tables only (the ones the kernels read in WinMeta: nitems, npitems, nlmb, ...)
enum SolvePath { SOLVE_UNFUSED, SOLVE_COMPACT, SOLVE_WIDE };      // lin_vis + lm_reduce + asm_items; host runs of lin_vis_lm; landmark blocks of lin_vis_lm_wide + asm_pairs_wide
enum MargPath { MARG_NONE, MARG_UNFUSED, MARG_WIDE };             // none: no visual factor is marginalised (window not full, no flag, or MARGIN_SECOND_NEW)
struct WinLow {
    int err; bool grouped, has_prior;
    bool dev_obs;                                     // the observations and inverse depths are filled on the device (fm_batch_fill), vis_obs is NULL
    int prior_n_out;
    bool obs_per_factor; int nobs_i, obsi_off;       // entries of the host-side observation table (wire format): one per run of factors with an identical (pts_i, velocity_i, td_i)
    int solve, marg;                                  // SolvePath, MargPath
    int nlist_s, nlist_m;                             // unfused solve / marginalisation: gather-list entries (emit_lists)
    int nrun, nrtile, rtile_off;                      // compact solve: host runs of lin_vis_lm, their tiles, the first tile's index
    int run_nt[NFR], run_slot[NFR];                   // per host frame: tiles of its run, the run's descriptor index (runs are ordered longest first)
};
static int chunk_count(int n, int chunk = ASM_CHUNK) { return (n + chunk - 1) / chunk; }
// columns of a visual factor's 12-double observation record (viwb.h): pts_i (0..2) pts_j (3..5) velocity_i (6,7) velocity_j (8,9) td_i (10) td_j (11)
static inline bool same_host_side(const double *a, const double *b) {      // bitwise (the wire format must reproduce the caller's table exactly)
    auto bits = [](const double *p) { unsigned long long v; memcpy(&v, p, sizeof v); return v; };
    return ((bits(a) ^ bits(b)) | (bits(a + 1) ^ bits(b + 1)) | (bits(a + 2) ^ bits(b + 2)) | (bits(a + 6) ^ bits(b + 6)) | (bits(a + 7) ^ bits(b + 7)) | (bits(a + 10) ^ bits(b + 10))) == 0;
}
static void split_obs(const double *o, double *hi, double *hj) { hi[0] = o[0]; hi[1] = o[1]; hi[2] = o[2]; hi[3] = o[6]; hi[4] = o[7]; hi[5] = o[10]; hj[0] = o[3]; hj[1] = o[4]; hj[2] = o[5]; hj[3] = o[8]; hj[4] = o[9]; hj[5] = o[11]; }

// Host runs of a compact fused window (kernels_fused.cuh, lin_vis_lm): per host frame, ascending, the landmarks it hosts in landmark order, cut into
// tiles of whole landmarks with at most LMB_FACTORS factors.  A landmark without factors joins the run of the lowest host frame, so that its outputs
// are still written.  A host's landmarks need not be consecutive: each run is a list.  visit(host, landmark, first factor, factor count, opens a tile)
// is called for every landmark, run by run, in run order.  vl / vi: the grouped factor table's landmarks and host frames.
template <typename F> static void host_runs(int nvis, const int *vl, const int *vi, int nlm, F visit) {
    static thread_local std::vector<int> first, cnt;
    first.assign(nlm > 0 ? nlm : 1, 0); cnt.assign(nlm > 0 ? nlm : 1, 0);
    int h0 = NFR;
    for (int i = 0; i < nvis; i++) { if (cnt[vl[i]]++ == 0) first[vl[i]] = i; h0 = std::min(h0, vi[i]); }
    for (int h = h0; h < NFR; h++) {
        int in_tile = 0; bool open = false;
        for (int k = 0; k < nlm; k++) {
            if ((cnt[k] ? vi[first[k]] : h0) != h) continue;
            const bool fresh = !open || in_tile + cnt[k] > LMB_FACTORS;
            if (fresh) { in_tile = 0; open = true; }
            in_tile += cnt[k];
            visit(h, k, first[k], cnt[k], fresh);
        }
    }
}

static void lower_count(const viwb_problem &p, int mf, bool allow_fused, bool dev_obs, WinMeta &m, WinLow &lo, int &out_mode) {
    memset(&m, 0, sizeof m); memset(&lo, 0, sizeof lo);
    lo.dev_obs = dev_obs;
    if (p.frame_count < 0 || p.frame_count > VIWB_WINDOW_SIZE || p.num_landmarks < 0 || p.num_landmarks > VIWB_MAX_LANDMARKS) { lo.err = 1; return; }
    if (p.num_vis < 0 || p.num_imu < 0 || p.num_wheel < 0 || p.num_plane < 0) { lo.err = 5; return; }            // counts are added up as size_t below
    if ((p.num_vis && (!p.vis_type || !p.vis_landmark || !p.vis_frame_i || !p.vis_frame_j || (!p.vis_obs && !dev_obs))) || (p.num_imu && (!p.imu_frame_i || !p.imu_frame_j || !p.imu_data)) ||
        (p.num_wheel && (!p.wheel_frame_i || !p.wheel_frame_j || !p.wheel_data)) || (p.num_plane && !p.plane_frame)) { lo.err = 5; return; }
    m.nlm = p.num_landmarks; m.frame_count = p.frame_count; m.nvis = p.num_vis; m.nimu = p.num_imu; m.nwheel = p.num_wheel; m.nplane = p.num_plane;
    for (int k = 0; k < 3; k++) m.G[k] = p.globals.G[k];
    for (int k = 0; k < 4; k++) m.S_vis[k] = p.globals.vis_sqrt_info[k];
    for (int k = 0; k < 3; k++) m.w_plane[k] = p.globals.plane_sqrt_info[k];
    m.huber = p.globals.huber_delta;
    lo.has_prior = p.prior && p.prior->valid;
    if (lo.has_prior && (p.prior->n <= 0 || p.prior->n > MAXPRI || p.prior->num_blocks <= 0 || p.prior->num_blocks > NB || !p.prior->J || !p.prior->r || !p.prior->x0)) { lo.err = 2; return; }
    if (lo.has_prior) {      // every kept block once, inside [0, n), no two blocks overlapping: prior_dx and the prior's assembly trust the column map
        unsigned seen_id = 0; unsigned char used[MAXPRI]; memset(used, 0, sizeof used);
        for (int i = 0; i < p.prior->num_blocks; i++) {
            const int bq = p.prior->block_id[i], idx = p.prior->block_idx[i];
            if (bq < 0 || bq >= NB || ((seen_id >> bq) & 1u)) { lo.err = 2; return; }
            seen_id |= 1u << bq;
            const int ms = blk_msize(bq);
            if (idx < 0 || idx + ms > p.prior->n) { lo.err = 2; return; }
            for (int k = 0; k < ms; k++) { if (used[idx + k]) { lo.err = 2; return; } used[idx + k] = 1; }
        }
    }
    // visual table checks + per-list counts
    int fcnt[NFR] = {0}, pcnt[NFR * NFR] = {0}, fcnt0[NFR] = {0}, pcnt0[NFR * NFR] = {0}, ncommon0 = 0;
    bool ref[NB]; for (int k = 0; k < NB; k++) ref[k] = false;
    bool seen[NB]; for (int k = 0; k < NB; k++) seen[k] = false;
    bool any_lm0 = false;
    lo.grouped = true;
    for (int i = 0; i < p.num_vis; i++) {
        const int t = p.vis_type[i], l = p.vis_landmark[i], fi = p.vis_frame_i[i], fj = p.vis_frame_j[i];
        if (t < 0 || t > 2 || l < 0 || l >= p.num_landmarks || fi < 0 || fi > p.frame_count || fj < 0 || fj > p.frame_count) { lo.err = 3; return; }
        if (i && l < p.vis_landmark[i - 1]) lo.grouped = false;
        if (t != 2 && fi == fj) { lo.err = 3; return; }       // a two-frame factor joins two different frames (estimator.cpp:1601-1603); the pair lists have no (a, a) slot
        if (t != 2) {
            ref[fi] = ref[fj] = true; fcnt[fi]++; fcnt[fj]++;
            const int a = fi < fj ? fi : fj, c = fi < fj ? fj : fi; pcnt[a * NFR + c]++;
            if (fi == 0) { fcnt0[fi]++; fcnt0[fj]++; pcnt0[a * NFR + c]++; seen[0] = seen[fj] = true; }
        }
        ref[BLK_EX0] = true; if (t != 0) ref[BLK_EX1] = true; ref[BLK_TD] = true;
        if (fi == 0) { any_lm0 = true; ncommon0++; seen[BLK_EX0] = true; if (t != 0) seen[BLK_EX1] = true; seen[BLK_TD] = true; }
    }
    {   // every factor of a landmark is hosted by the landmark's start frame (estimator.cpp:1595-1597): lm_reduce adds the host blocks of a landmark into ONE row of W
        short host[VIWB_MAX_LANDMARKS];
        for (int k = 0; k < p.num_landmarks; k++) host[k] = -1;
        for (int i = 0; i < p.num_vis; i++) { short &h = host[p.vis_landmark[i]]; if (h < 0) h = (short)p.vis_frame_i[i]; else if (h != p.vis_frame_i[i]) { lo.err = 3; return; } }
    }
    if (lo.has_prior) for (int i = 0; i < p.prior->num_blocks; i++) ref[p.prior->block_id[i]] = true;
    for (int i = 0; i < p.num_imu; i++) { const int a = p.imu_frame_i[i], c = p.imu_frame_j[i]; if (a < 0 || a > p.frame_count || c < 0 || c > p.frame_count) { lo.err = 4; return; } ref[a] = ref[BLK_SB0 + a] = ref[c] = ref[BLK_SB0 + c] = true; }
    for (int i = 0; i < p.num_wheel; i++) { const int a = p.wheel_frame_i[i], c = p.wheel_frame_j[i]; if (a < 0 || a > p.frame_count || c < 0 || c > p.frame_count) { lo.err = 4; return; } ref[a] = ref[c] = ref[BLK_EXW] = ref[BLK_SX] = ref[BLK_SY] = ref[BLK_SW] = ref[BLK_TDW] = true; }
    for (int i = 0; i < p.num_plane; i++) { const int a = p.plane_frame[i]; if (a < 0 || a > p.frame_count) { lo.err = 4; return; } ref[a] = ref[BLK_EXW] = ref[BLK_PR] = ref[BLK_PZ] = true; }
    // active blocks (Program::RemoveFixedBlocks) and compact columns
    // Column order = elimination order of the dense Cholesky.  The speed-bias blocks come first, newest frame first: each couples
    // only with its neighbour in the IMU chain and two poses, so the factor keeps a narrow profile there (a "skyline": row i is
    // stored from its first structurally non-zero column efirst[i]; Cholesky never fills outside that envelope).
    int col = 0;
    bool active[NB];
    for (int k = 0; k < NB; k++) {
        m.flags[k] = p.block_flags[k] & 3u; m.mask[k] = p.subset_mask[k];
        active[k] = (p.block_flags[k] & VIWB_BLOCK_PRESENT) && !(p.block_flags[k] & VIWB_BLOCK_CONSTANT) && ref[k];
        m.tcol[k] = -1;
    }
    for (int f = VIWB_WINDOW_SIZE; f >= 0; f--) { const int k = BLK_SB0 + f; if (active[k]) { m.tcol[k] = (short)col; col += blk_tsize(k); } }
    for (int k = 0; k < NB; k++) if (active[k] && m.tcol[k] < 0) { m.tcol[k] = (short)col; col += blk_tsize(k); }
    m.nf = col;
    {   // symbolic envelope: every factor makes the blocks it touches a clique
        int first_blk[NB];
        for (int k = 0; k < NB; k++) first_blk[k] = m.tcol[k];                 // the diagonal block itself
        auto clique = [&](const int *blks, int n) {
            int lo = TFIX;
            for (int q = 0; q < n; q++) if (blks[q] >= 0 && m.tcol[blks[q]] >= 0 && m.tcol[blks[q]] < lo) lo = m.tcol[blks[q]];
            for (int q = 0; q < n; q++) if (blks[q] >= 0 && m.tcol[blks[q]] >= 0 && lo < first_blk[blks[q]]) first_blk[blks[q]] = lo;
        };
        if (lo.has_prior) { int bl[NB]; for (int i = 0; i < p.prior->num_blocks; i++) bl[i] = p.prior->block_id[i]; clique(bl, p.prior->num_blocks); }
        for (int i = 0; i < p.num_imu; i++) { const int a = p.imu_frame_i[i], c = p.imu_frame_j[i]; const int bl[4] = {a, BLK_SB0 + a, c, BLK_SB0 + c}; clique(bl, 4); }
        for (int i = 0; i < p.num_wheel; i++) { const int bl[7] = {p.wheel_frame_i[i], p.wheel_frame_j[i], BLK_EXW, BLK_SX, BLK_SY, BLK_SW, BLK_TDW}; clique(bl, 7); }
        for (int i = 0; i < p.num_plane; i++) { const int bl[4] = {p.plane_frame[i], BLK_EXW, BLK_PR, BLK_PZ}; clique(bl, 4); }
        if (p.num_vis > 0) {       // after the landmark elimination the visual subspace (all observed poses, ex0, ex1, td) is dense
            int bl[NFR + 3], n = 0;
            for (int f = 0; f <= VIWB_WINDOW_SIZE; f++) if (ref[f]) bl[n++] = f;
            bl[n++] = BLK_EX0; bl[n++] = BLK_EX1; bl[n++] = BLK_TD;
            clique(bl, n);
        }
        int es = 0;
        for (int k = 0; k < NB; k++) if (m.tcol[k] >= 0) for (int r = 0; r < blk_tsize(k); r++) { const int i = m.tcol[k] + r; m.efirst[i] = (short)first_blk[k]; es += i - first_blk[k] + 1; }
        m.esize = es;
    }
    m.has_common = (m.tcol[BLK_EX0] >= 0 || m.tcol[BLK_EX1] >= 0 || m.tcol[BLK_TD] >= 0) ? 1 : 0;
    // marginalisation plan (estimator.cpp:1666-1893)
    m.margin_flag = -1; out_mode = 2; lo.prior_n_out = 0;
    if (mf >= 0 && p.frame_count == VIWB_WINDOW_SIZE) {
        if (mf == VIWB_MARGIN_OLD) {
            if (lo.has_prior) for (int i = 0; i < p.prior->num_blocks; i++) seen[p.prior->block_id[i]] = true;
            for (int i = 0; i < p.num_imu; i++) if (p.imu_frame_i[i] == 0 && p.imu_frame_j[i] == 1) seen[0] = seen[BLK_SB0] = seen[1] = seen[BLK_SB0 + 1] = true;
            for (int i = 0; i < p.num_wheel; i++) if (p.wheel_frame_i[i] == 0 && p.wheel_frame_j[i] == 1) seen[0] = seen[1] = seen[BLK_EXW] = seen[BLK_SX] = seen[BLK_SY] = seen[BLK_SW] = seen[BLK_TDW] = true;
            for (int i = 0; i < p.num_plane; i++) if (p.plane_frame[i] == 0) seen[0] = seen[BLK_EXW] = seen[BLK_PR] = seen[BLK_PZ] = true;
            if (seen[0] || seen[BLK_SB0] || any_lm0) { m.margin_flag = 0; out_mode = 0; }
        } else {
            for (int k = 0; k < NB; k++) seen[k] = false;
            bool has9 = false;
            if (lo.has_prior) for (int i = 0; i < p.prior->num_blocks; i++) { seen[p.prior->block_id[i]] = true; if (p.prior->block_id[i] == VIWB_WINDOW_SIZE - 1) has9 = true; }
            if (has9) { m.margin_flag = 1; out_mode = 0; } else out_mode = lo.has_prior ? 1 : 2;
        }
        if (m.margin_flag >= 0) {
            int nn = 0;
            for (int k = 0; k < NB; k++) if (seen[k]) { m.flags[k] |= 4u; const bool drop = m.margin_flag == 0 ? (k == 0 || k == BLK_SB0) : (k == VIWB_WINDOW_SIZE - 1); if (!drop) nn += blk_msize(k); }
            lo.prior_n_out = nn;
        }
    }
    // wire format: runs of factors sharing one host-side observation (a grouped table: one run per landmark, estimator.cpp:1595-1597 takes
    // pts_i / velocity_i / td_i from the landmark's first observation for every factor); an ungrouped table keeps one entry per factor
    // (assumed here -- the plan never reads the observations --, verified when lower_fill copies them; a table that breaks it is rebuilt with one entry per factor)
    lo.obs_per_factor = !lo.grouped; lo.nobs_i = lo.grouped ? p.num_landmarks : p.num_vis;
    // the paths (kernels_fused.cuh).  A regular table -- grouped, <= LMB_FACTORS factors per landmark, at most two factors per (landmark, observer),
    // consecutive -- takes the fused path where it has pair chunks: compact records (host runs) unless ex0 / ex1 / td are active, wide records
    // otherwise; the marginalisation of frame 0 always takes wide records.  Decided per window, so that a window takes the same path -- and gives
    // the same bits -- whatever else the batch holds.  nlmb: landmark blocks of lin_vis_lm_wide (whole landmarks, <= LMB_FACTORS factors)
    bool regular = lo.grouped;
    int nlmb = 0;
    for (int k = 0, i = 0, in_blk = 0; k < p.num_landmarks && regular; k++) {
        int cnt = 0, seenj[NFR], ndup[NFR];
        for (int q = 0; q < NFR; q++) { seenj[q] = -2; ndup[q] = 0; }
        for (; i < p.num_vis && p.vis_landmark[i] == k; i++, cnt++) {
            if (p.vis_type[i] == 2) continue;
            const int fj = p.vis_frame_j[i];
            if (ndup[fj] == 0) { ndup[fj] = 1; seenj[fj] = i; }
            else if (ndup[fj] == 1 && seenj[fj] == i - 1) ndup[fj] = 2;
            else regular = false;
        }
        if (cnt > LMB_FACTORS) regular = false;
        if (k == 0 || in_blk + cnt > LMB_FACTORS) { nlmb++; in_blk = 0; }
        in_blk += cnt;
    }
    // pair chunks: one group per frame pair; with wide records the one-frame factors (which carry ex0 / ex1 / td columns) form the "pairs" (host, host)
    int npit = 0, nmpit = 0, nxrec = 0, two0 = 0, scnt[NFR] = {0};
    if (m.has_common) for (int i = 0; i < p.num_vis; i++) if (p.vis_type[i] == 2) scnt[p.vis_frame_i[i]]++;
    for (int a = 0; a < NFR * NFR; a++) { nxrec += pcnt[a]; npit += chunk_count(pcnt[a], PAIR_CHUNK); two0 += pcnt0[a]; nmpit += chunk_count(pcnt0[a], PAIR_CHUNK); }
    for (int a = 0; a < NFR; a++) { nxrec += scnt[a]; npit += chunk_count(scnt[a], PAIR_CHUNK); }
    nmpit += chunk_count(ncommon0 - two0, PAIR_CHUNK);
    const bool fused = allow_fused && regular && npit > 0, mfused = allow_fused && regular && m.margin_flag == 0 && nmpit > 0;
    lo.solve = !fused ? SOLVE_UNFUSED : m.has_common ? SOLVE_WIDE : SOLVE_COMPACT;
    lo.marg = m.margin_flag != 0 ? MARG_NONE : mfused ? MARG_WIDE : MARG_UNFUSED;
    m.fused = fused; m.mfused = mfused;
    // the sizes of the chosen paths' tables; lower_fill builds them
    auto list_sizes = [](const int *fc, const int *pc, int ncom, int &nlist, int &nitems) {      // emit_lists: frame lists, pair lists, common list
        auto add = [&](int n) { nlist += n; nitems += chunk_count(n); };
        for (int a = 0; a < NFR; a++) add(fc[a]);
        for (int a = 0; a < NFR * NFR; a++) add(pc[a]);
        add(ncom);
    };
    if (lo.solve == SOLVE_UNFUSED) list_sizes(fcnt, pcnt, m.has_common ? p.num_vis : 0, lo.nlist_s, m.nitems);
    if (lo.solve == SOLVE_COMPACT) {      // the pairs' products are formed per host run, no record is stored
        m.npitems = npit;
        host_runs(p.num_vis, p.vis_landmark, p.vis_frame_i, p.num_landmarks, [&](int h, int, int, int, bool fresh) { if (fresh) { if (lo.run_nt[h]++ == 0) lo.nrun++; lo.nrtile++; } });
    }
    if (lo.solve == SOLVE_WIDE) { m.npitems = npit; m.nxrec = nxrec; }
    if (lo.marg == MARG_UNFUSED) list_sizes(fcnt0, pcnt0, ncommon0, lo.nlist_m, m.nmitems);
    if (lo.marg == MARG_WIDE) { m.nmpitems = nmpit; m.nmxrec = ncommon0; }
    if (lo.solve == SOLVE_WIDE || lo.marg == MARG_WIDE) m.nlmb = nlmb;
}

// ---- phase 3: fill this window's slices of the (pinned) staging arrays; every offset is final
struct HostArrays {      // the input arrays' views in the staging slab (batch_build's slab table sets them)
    WinMeta *meta; PriorDev *prior; int *vis_code, *vis_lm, *vis_oi; double *obs_i, *obs_j; int *lm_win, *lm_fptr; double *x_fix; int *fm_off;
    AsmItem *items; int *asm_list; int *imu_fi, *imu_fj, *imu_win, *wheel_fi, *wheel_fj, *wheel_win, *plane_f, *plane_win;
    double *imu_data, *wheel_data, *prior_J, *prior_r, *prior_x0, *x_init; WinWork *work;
    int nitems_solve_total, meta_count;
    int *vis_pos; LmbDesc *lmb_desc; AsmItem *pitems; int *mvis_pos; AsmItem *mpitems;
    RunDesc *run_desc; RunTile *run_tile; int *run_f, *run_lm;
    unsigned char *obs_viol;        // [B] host only: set by lower_fill when a grouped table does not share one host-side observation per landmark
};
static void emit_lists(const int *type, const int *fi, const int *fj, int nvis, bool only_host0, int has_common, int w, AsmItem *items, int *list) {
    // counting sort of the (factor, role) entries into frame lists, pair lists and the common list, then chunking
    int fcnt[NFR] = {0}, pcnt[NFR * NFR] = {0}, ncom = 0;
    for (int i = 0; i < nvis; i++) {
        if (only_host0 && fi[i] != 0) continue;
        if (type[i] != 2) { fcnt[fi[i]]++; fcnt[fj[i]]++; const int a = fi[i] < fj[i] ? fi[i] : fj[i], c = fi[i] < fj[i] ? fj[i] : fi[i]; pcnt[a * NFR + c]++; }
        ncom++;
    }
    int foff[NFR], poff[NFR * NFR], pos = 0;
    for (int a = 0; a < NFR; a++) { foff[a] = pos; pos += fcnt[a]; }
    for (int a = 0; a < NFR * NFR; a++) { poff[a] = pos; pos += pcnt[a]; }
    const int coff = pos;
    int fpos[NFR], ppos[NFR * NFR], cpos = coff;
    memcpy(fpos, foff, sizeof fpos); memcpy(ppos, poff, sizeof ppos);
    for (int i = 0; i < nvis; i++) {
        if (only_host0 && fi[i] != 0) continue;
        if (type[i] != 2) {
            list[fpos[fi[i]]++] = (i << 1) | 0; list[fpos[fj[i]]++] = (i << 1) | 1;
            const int a = fi[i] < fj[i] ? fi[i] : fj[i], c = fi[i] < fj[i] ? fj[i] : fi[i];
            list[ppos[a * NFR + c]++] = (i << 1) | (fi[i] == a ? 0 : 1);
        }
        if (has_common) list[cpos++] = i << 1;
    }
    int ni = 0;
    auto emit = [&](int kind, int a, int c, int off, int cnt) {
        for (int c0 = 0, ph = 0; c0 < cnt; c0 += ASM_CHUNK, ph++) {
            AsmItem &it = items[ni++];
            it.kind = kind; it.win = w; it.a = a; it.b = c; it.lo = off + c0; it.hi = off + std::min(cnt, c0 + (int)ASM_CHUNK); it.phase = ph; it.has_common = has_common;
        }
    };
    for (int a = 0; a < NFR; a++) emit(ITEM_FRAME, a, a, foff[a], fcnt[a]);
    for (int a = 0; a < NFR; a++) for (int c = a + 1; c < NFR; c++) emit(ITEM_PAIR, a, c, poff[a * NFR + c], pcnt[a * NFR + c]);
    if (has_common) emit(ITEM_COMMON, 0, 0, coff, ncom);
}

static void lower_fill(const viwb_problem &p, const double *state, int w, const WinMeta &m, const WinLow &lo, const HostArrays &h, double init_radius) {
    h.meta[w] = m;
    // visual factors grouped by landmark
    // (the per-factor type / frames / duplicate code travel as ONE code word and are unpacked on the device: the tables below are host scratch)
    static thread_local std::vector<int> scratch; static thread_local std::vector<unsigned char> scratch_d;
    scratch.resize((size_t)3 * p.num_vis + 1); scratch_d.assign((size_t)p.num_vis + 1, 0);
    int *vt = scratch.data(), *vi = vt + p.num_vis, *vj = vi + p.num_vis, *vl = h.vis_lm + m.vis_off;
    unsigned char *vd = scratch_d.data();
    double *oj = h.obs_j + (size_t)m.vis_off * 6, *oi = h.obs_i + (size_t)lo.obsi_off * 6;
    int *voi = h.vis_oi + m.vis_off;
    if (lo.grouped) {
        memcpy(vt, p.vis_type, sizeof(int) * p.num_vis); memcpy(vl, p.vis_landmark, sizeof(int) * p.num_vis);
        memcpy(vi, p.vis_frame_i, sizeof(int) * p.num_vis); memcpy(vj, p.vis_frame_j, sizeof(int) * p.num_vis);
        int run = -1;
        for (int i = 0; i < p.num_vis; i++) {
            if (lo.dev_obs) { if (i == 0 || vl[i] != vl[i - 1]) run++; voi[i] = lo.obsi_off + run; continue; }      // one host side per landmark, filled on the device
            const double *o = p.vis_obs + (size_t)i * 12;
            double hi[6];
            split_obs(o, hi, oj + (size_t)i * 6);
            if (lo.obs_per_factor) { memcpy(oi + (size_t)i * 6, hi, sizeof hi); voi[i] = lo.obsi_off + i; continue; }
            if (i == 0 || vl[i] != vl[i - 1]) { run++; memcpy(oi + (size_t)run * 6, hi, sizeof hi); }
            else if (!same_host_side(o, o - 12)) h.obs_viol[w] = 1;          // two factors of one landmark with different host-side observations: the caller of lower_fill rebuilds
            voi[i] = lo.obsi_off + run;
        }
    } else {
        std::vector<int> order(p.num_vis);
        for (int i = 0; i < p.num_vis; i++) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](int a, int c) { return p.vis_landmark[a] < p.vis_landmark[c]; });
        for (int i = 0; i < p.num_vis; i++) {
            const int sidx = order[i]; vt[i] = p.vis_type[sidx]; vl[i] = p.vis_landmark[sidx]; vi[i] = p.vis_frame_i[sidx]; vj[i] = p.vis_frame_j[sidx];
            split_obs(p.vis_obs + (size_t)sidx * 12, oi + (size_t)i * 6, oj + (size_t)i * 6); voi[i] = lo.obsi_off + i;
        }
    }
    // landmark -> factor ranges (global factor indices)
    { int *fp = h.lm_fptr + m.lm_off; int run = m.vis_off, i = 0;
      for (int k = 0; k < p.num_landmarks; k++) { fp[k] = run; while (i < p.num_vis && vl[i] == k) { i++; run++; } h.lm_win[m.lm_off + k] = w; } }
    // the tables of the window's paths (lower_count sized exactly these)
    // pair_tables: frame-pair order of the X records (counting sort by (host, observer); the one-frame factors of WIDE records form the "pair" (host, host)),
    // pair chunks; for the solver (all factors) and for the marginalisation of frame 0 (the factors hosted there).  vp: each factor's record slot
    // (nullptr: compact solver windows, whose records are never stored); first_item: per pair (host * NFR + observer) its first chunk, -1: none
    auto pair_tables = [&](bool marg, int *vp, AsmItem *pit, int base, int wide, int *first_item) {
        int pcnt[NFR * NFR] = {0}, poff[NFR * NFR];
        for (int i = 0; i < p.num_vis; i++) {
            if (marg && vi[i] != 0) continue;
            if (vt[i] != 2) pcnt[vi[i] * NFR + vj[i]]++; else if (wide) pcnt[vi[i] * NFR + vi[i]]++;
        }
        int pos = 0, ni = 0;
        for (int a = 0; a < NFR * NFR; a++) {
            poff[a] = pos;
            first_item[a] = pcnt[a] ? ni : -1;
            for (int c0 = 0, ph = 0; c0 < pcnt[a]; c0 += PAIR_CHUNK, ph++) {
                AsmItem &it = pit[ni++];
                it.kind = ITEM_PAIR; it.win = w; it.a = a / NFR; it.b = a % NFR; it.lo = pos + c0; it.hi = pos + std::min(pcnt[a], c0 + (int)PAIR_CHUNK); it.phase = ph; it.has_common = wide; it.base = base;
            }
            pos += pcnt[a];
        }
        if (vp) for (int i = 0; i < p.num_vis; i++) {
            if (marg && vi[i] != 0) { vp[i] = -1; continue; }
            if (vt[i] != 2) vp[i] = poff[vi[i] * NFR + vj[i]]++; else if (wide) vp[i] = poff[vi[i] * NFR + vi[i]]++; else vp[i] = -1;
        }
    };
    auto landmark_table = [&]() {      // landmark blocks of lin_vis_lm_wide (the wide solve and the wide marginalisation share them)
        LmbDesc *ld = h.lmb_desc + m.lmb_off;
        for (int k = 0, i = 0, nb = 0; k < p.num_landmarks; k++) {
            const int first = i;
            while (i < p.num_vis && vl[i] == k) i++;
            if (k == 0 || ld[nb - 1].nf + (i - first) > LMB_FACTORS) { LmbDesc &d = ld[nb++]; memset(&d, 0, sizeof d); d.win = w; d.k0 = m.lm_off + k; d.f0 = m.vis_off + first; }
            ld[nb - 1].k1 = m.lm_off + k + 1;           // the open block ends after this landmark
            ld[nb - 1].nf += i - first;
        }
    };
    int pfirst[NFR * NFR];
    switch (lo.solve) {
    case SOLVE_UNFUSED: emit_lists(vt, vi, vj, p.num_vis, false, m.has_common, w, h.items + m.item_off, h.asm_list + m.list_off); break;
    case SOLVE_WIDE: pair_tables(false, h.vis_pos + m.vis_off, h.pitems + m.pitem_off, m.xrec_off, 1, pfirst); landmark_table(); break;
    case SOLVE_COMPACT: {      // pair chunks without records; host runs: descriptors (at their slot in the longest-first order), tiles, factor and landmark lists in run order
        pair_tables(false, nullptr, h.pitems + m.pitem_off, m.xrec_off, 0, pfirst);
        int *rf = h.run_f + m.vis_off, *rl = h.run_lm + 2 * (size_t)m.lm_off;
        RunTile *rt = h.run_tile + lo.rtile_off;
        int nfac = 0, nlmk = 0, ntl = 0, cur = -1;
        host_runs(p.num_vis, vl, vi, p.num_landmarks, [&](int hf, int k, int first, int cnt, bool fresh) {
            if (hf != cur) {
                RunDesc &d = h.run_desc[lo.run_slot[hf]]; memset(&d, 0, sizeof d);
                d.win = w; d.host = hf; d.t0 = lo.rtile_off + ntl; d.ntile = lo.run_nt[hf];
                for (int j = 0; j < NFR; j++) d.pfirst[j] = pfirst[hf * NFR + j] >= 0 ? m.pitem_off + pfirst[hf * NFR + j] : -1;
                cur = hf;
            }
            if (fresh) { RunTile &t = rt[ntl++]; t.l0 = m.lm_off + nlmk; t.nl = 0; t.f0 = m.vis_off + nfac; t.nf = 0; }
            RunTile &t = rt[ntl - 1];
            rl[2 * nlmk] = m.lm_off + k; rl[2 * nlmk + 1] = t.nf; nlmk++; t.nl++;
            for (int q = 0; q < cnt; q++) rf[nfac++] = m.vis_off + first + q;
            t.nf += cnt;
        });
        break;
    }
    }
    switch (lo.marg) {      // (MARG_NONE: no table)
    case MARG_UNFUSED: emit_lists(vt, vi, vj, p.num_vis, true, 1, w, h.items + h.nitems_solve_total + m.mitem_off, h.asm_list + m.mlist_off); break;
    case MARG_WIDE: pair_tables(true, h.mvis_pos + m.vis_off, h.mpitems + m.mpitem_off, m.mxrec_off, 1, pfirst); if (lo.solve != SOLVE_WIDE) landmark_table(); break;
    }
    if (m.fused || m.mfused) {      // duplicate codes (two factors of one landmark observed from the same frame: left and right camera, consecutive)
        for (int i = 0; i < p.num_vis; i++) {
            if (vt[i] == 2) continue;
            if (i > 0 && vt[i - 1] != 2 && vl[i - 1] == vl[i] && vj[i - 1] == vj[i]) { vd[i - 1] = 1; vd[i] = 2; }
        }
    }
    { int *vc = h.vis_code + m.vis_off; for (int i = 0; i < p.num_vis; i++) vc[i] = vt[i] | (vi[i] << 2) | (vj[i] << 6) | ((int)vd[i] << 10); }

    // small factors
    for (int i = 0; i < p.num_imu; i++) { h.imu_fi[m.imu_off + i] = p.imu_frame_i[i]; h.imu_fj[m.imu_off + i] = p.imu_frame_j[i]; h.imu_win[m.imu_off + i] = w; }
    if (p.num_imu) memcpy(h.imu_data + (size_t)m.imu_off * 287, p.imu_data, sizeof(double) * 287 * p.num_imu);
    for (int i = 0; i < p.num_wheel; i++) { h.wheel_fi[m.wheel_off + i] = p.wheel_frame_i[i]; h.wheel_fj[m.wheel_off + i] = p.wheel_frame_j[i]; h.wheel_win[m.wheel_off + i] = w; }
    if (p.num_wheel) memcpy(h.wheel_data + (size_t)m.wheel_off * 78, p.wheel_data, sizeof(double) * 78 * p.num_wheel);
    for (int i = 0; i < p.num_plane; i++) { h.plane_f[m.plane_off + i] = p.plane_frame[i]; h.plane_win[m.plane_off + i] = w; }
    // prior
    if (m.prior_idx >= 0) {
        const viwb_prior &pr = *p.prior; PriorDev &pd = h.prior[m.prior_idx];
        memcpy(h.prior_J + pd.J_off, pr.J, sizeof(double) * pr.n * pr.n); memcpy(h.prior_r + pd.r_off, pr.r, sizeof(double) * pr.n);
        memcpy(h.prior_x0 + pd.x0_off, pr.x0, sizeof(double) * SFIX);
    }
    if (lo.dev_obs) { memcpy(h.x_fix + (size_t)SFIX * w, state, sizeof(double) * SFIX); h.fm_off[w] = m.state_off; h.fm_off[h.meta_count + w] = m.lm_off; }
    else memcpy(h.x_init + m.state_off, state, sizeof(double) * (SFIX + p.num_landmarks));
    WinWork &ww = h.work[w]; memset(&ww, 0, sizeof ww);
    ww.status = ST_RUNNING; ww.phase = PH_INIT; ww.first = 1; ww.radius = init_radius; ww.mu = 1e-8; ww.mu_lin = 1e-8; ww.term = VIWB_NO_CONVERGENCE;
}

template <typename F> static void parallel_for(int n, F f) {
    // host threads of the lowering: VIWB_HOST_THREADS (a caller that drives several contexts from several threads divides the cores among them), else
    // all hardware threads up to 16
    const char *env_nt = getenv("VIWB_HOST_THREADS");
    const int cap = (env_nt && atoi(env_nt) > 0) ? atoi(env_nt) : 16;
    int nt = (int)std::thread::hardware_concurrency(); if (nt > cap) nt = cap; if (nt < 1) nt = 1; if (nt > n / 8) nt = n / 8;
    if (nt <= 1) { for (int i = 0; i < n; i++) f(i); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++) th.emplace_back([=]() { for (int i = t; i < n; i += nt) f(i); });
    for (auto &t : th) t.join();
}

static void fm_fill_batch(viwb_features *fs, const viwb_batch *b);
// from: the windows' visual tables are index tables rebuilt from these lists (viwb_features_batch_create), their observations and landmark states are
// filled from the lists on the device after the upload, which leaves them out
static int batch_build(viwb_context *ctx, int B, const viwb_problem *problems, const double *const *states,
                       const viwb_options *options, const int32_t *margin_flags, viwb_batch **out, bool use_cached = false, bool obs_per_factor = false,
                       viwb_features *from = nullptr) {
    bind_device(ctx);
    if (B <= 0 || !problems || !states) return fail(ctx, VIWB_ERR_INVALID, "empty batch");
    const double t_start = now_ms();
    viwb_batch *b = new viwb_batch();
    b->B = B; b->any_marg = false; b->algorithmic_bytes = 0; b->arena_cached = false; b->out_bytes = 0; b->prior_nmax = 0; b->work_init_dev = nullptr;
    b->fs = nullptr; b->fs_gen = 0; b->x_fix = nullptr; b->fm_off = nullptr;
    const bool dev_obs = from != nullptr;
    viwb_options defopt; viwb_default_options(&defopt);
    const viwb_options *opt = options ? options : &defopt;
    b->max_iter = opt->max_num_iterations;
    b->max_time = opt->max_solver_time_in_seconds;
    BatchDev &bd = b->bd; memset(&bd, 0, sizeof bd);
    bd.B = B; opts_from(opt, bd.opt);
    b->meta.resize(B); b->out_mode.assign(B, 2); b->in_prior.resize(B); b->state_sizes.resize(B); b->prior_n.assign(B, 0);
    std::vector<WinLow> low(B);
    // ---- phase 1 (parallel): sizes and plans
    const bool allow_fused = getenv("VIWB_NO_FUSED") == nullptr;      // read once per build: every window of the batch is planned under the same switch
    parallel_for(B, [&](int w) { lower_count(problems[w], margin_flags ? margin_flags[w] : -1, allow_fused, dev_obs, b->meta[w], low[w], b->out_mode[w]); });
    const double t_counted = now_ms();
    if (obs_per_factor) for (int w = 0; w < B; w++) { low[w].obs_per_factor = true; low[w].nobs_i = problems[w].num_vis < 0 ? 0 : problems[w].num_vis; }
    for (int w = 0; w < B; w++) if (low[w].err) { const int e = low[w].err; batch_free(ctx, b); return fail(ctx, VIWB_ERR_INVALID, e == 1 ? "bad frame_count / num_landmarks" : e == 2 ? "bad prior" : e == 3 ? "bad visual factor table" : e == 5 ? "negative factor count or missing table" : "bad factor frame index"); }
    for (const WinLow &lo : low) {
        bd.n_unfused += lo.solve == SOLVE_UNFUSED; bd.n_fused_compact += lo.solve == SOLVE_COMPACT; bd.n_fused_wide += lo.solve == SOLVE_WIDE;
        bd.n_munfused += lo.marg == MARG_UNFUSED; bd.n_mfused += lo.marg == MARG_WIDE;
    }
    // host runs, longest first (a counting sort by tile count): every window's long run (its frame-0 run, on the bench's windows) starts in the first
    // waves instead of forming the tail
    size_t nrun = 0, nrtile = 0;
    {
        int maxt = 0;
        for (int w = 0; w < B; w++) for (int f = 0; f < NFR; f++) maxt = std::max(maxt, low[w].run_nt[f]);
        std::vector<size_t> start((size_t)maxt + 2, 0);
        for (int w = 0; w < B; w++) for (int f = 0; f < NFR; f++) if (low[w].run_nt[f]) start[maxt - low[w].run_nt[f] + 1]++;
        for (int t = 1; t <= maxt + 1; t++) start[t] += start[t - 1];
        for (int w = 0; w < B; w++) {
            WinLow &lo = low[w];
            lo.rtile_off = (int)nrtile; nrtile += lo.nrtile; nrun += lo.nrun;
            for (int f = 0; f < NFR; f++) if (lo.run_nt[f]) lo.run_slot[f] = (int)start[maxt - lo.run_nt[f]]++;
        }
    }
    // factorisation plans (kernels_solve.cuh): one per distinct envelope, shared by the windows that have it -- the plan is a function of the
    // envelope alone, so a window is factored the same way whatever else the batch holds
    std::vector<std::vector<int>> plans;
    size_t nplan = 0;
    {
        std::map<std::vector<short>, int> env_plan;
        std::vector<int> env_of(B), env_win;
        for (int w = 0; w < B; w++) {
            const WinMeta &m = b->meta[w];
            auto ins = env_plan.emplace(std::vector<short>(m.efirst, m.efirst + m.nf), (int)env_win.size());
            if (ins.second) env_win.push_back(w);
            env_of[w] = ins.first->second;
        }
        plans.resize(env_win.size());
        parallel_for((int)env_win.size(), [&](int e) { const WinMeta &m = b->meta[env_win[e]]; chol_plan_build(m.efirst, m.nf, plans[e]); });
        std::vector<int> off(plans.size());
        for (size_t e = 0; e < plans.size(); e++) { off[e] = (int)nplan; nplan += plans[e].size(); }
        for (int w = 0; w < B; w++) b->meta[w].plan_off = off[env_of[w]];
    }
    // ---- phase 2: offsets
    size_t nlmb = 0, npit = 0, nxr = 0, nmpit = 0, nmxr = 0;      // nxr / nmxr: record regions in DOUBLES (solver / marginalisation share one buffer)
    size_t nobsi = 0;
    size_t nstate = 0, nvis = 0, nlm = 0, nimu = 0, nwheel = 0, nplane = 0, nlist = 0, nit_s = 0, nit_m = 0, npri = 0, npJ = 0, npr = 0;
    for (int w = 0; w < B; w++) {
        const viwb_problem &p = problems[w]; WinMeta &m = b->meta[w]; const WinLow &lo = low[w];
        m.state_off = (int)nstate; nstate += SFIX + p.num_landmarks; b->state_sizes[w] = SFIX + p.num_landmarks;
        m.vis_off = (int)nvis; nvis += p.num_vis; m.lm_off = (int)nlm; nlm += p.num_landmarks;
        low[w].obsi_off = (int)nobsi; nobsi += lo.nobs_i;
        m.imu_off = (int)nimu; nimu += p.num_imu; m.wheel_off = (int)nwheel; nwheel += p.num_wheel; m.plane_off = (int)nplane; nplane += p.num_plane;
        m.item_off = (int)nit_s; nit_s += m.nitems; m.list_off = (int)nlist; nlist += lo.nlist_s;
        m.prior_idx = lo.has_prior ? (int)npri++ : -1;
        m.lmb_off = (int)nlmb; nlmb += m.nlmb; m.pitem_off = (int)npit; npit += m.npitems; m.xrec_off = (int)nxr; nxr += (size_t)m.nxrec * XL<true>::REC;      // (only wide solver windows store records)
        m.mpitem_off = (int)nmpit; nmpit += m.nmpitems; m.mxrec_off = (int)nmxr; nmxr += (size_t)m.nmxrec * XL<true>::REC;
        b->prior_n[w] = lo.prior_n_out; if (m.margin_flag >= 0) b->any_marg = true;
        b->prior_nmax = std::max(b->prior_nmax, lo.prior_n_out);
        b->algorithmic_bytes += window_algorithmic_bytes(p, opt->max_num_iterations);
    }
    for (int w = 0; w < B; w++) { WinMeta &m = b->meta[w]; m.mitem_off = (int)nit_m; nit_m += m.nmitems; m.mlist_off = (int)nlist; nlist += low[w].nlist_m; }
    if (nxr > 0x7fffffff || nmxr > 0x7fffffff || nstate > 0x7fffffff || nvis * 12 > 0x7fffffffull * 4 || nlist > 0x7fffffff || nplan > 0x7fffffff) { batch_free(ctx, b); return fail(ctx, VIWB_ERR_INVALID, "batch too large"); }
    std::vector<PriorDev> priors(npri);
    for (int w = 0; w < B; w++) if (b->meta[w].prior_idx >= 0) {
        const viwb_prior &pr = *problems[w].prior; PriorDev &pd = priors[b->meta[w].prior_idx]; memset(&pd, 0, sizeof pd);
        pd.n = pr.n; pd.nb = pr.num_blocks;
        for (int i = 0; i < pr.num_blocks; i++) { pd.block_id[i] = pr.block_id[i]; pd.block_idx[i] = pr.block_idx[i]; }
        pd.J_off = (int)npJ; npJ += (size_t)pr.n * pr.n; pd.r_off = (int)npr; npr += pr.n; pd.x0_off = (int)(SFIX * (size_t)b->meta[w].prior_idx);
        HostPrior &hp = b->in_prior[w]; hp.valid = 1; hp.n = pr.n; hp.nb = pr.num_blocks;
        memcpy(hp.block_id, pd.block_id, sizeof hp.block_id); memcpy(hp.block_idx, pd.block_idx, sizeof hp.block_idx);
        if (b->out_mode[w] == 1) { hp.x0.assign(pr.x0, pr.x0 + SFIX); hp.J.assign(pr.J, pr.J + (size_t)pr.n * pr.n); hp.r.assign(pr.r, pr.r + pr.n); }
    }
    bd.nvis_total = (int)nvis; bd.nlm_total = (int)nlm; bd.nimu_total = (int)nimu; bd.nwheel_total = (int)nwheel; bd.nplane_total = (int)nplane; bd.nprior = (int)npri;
    bd.nitems_solve = (int)nit_s; bd.nitems_marg = (int)nit_m;
    bd.nlmb_total = (int)nlmb; bd.npitems_total = (int)npit; bd.nmpitems_total = (int)nmpit; bd.nrun_total = (int)nrun;
    bd.pitems_max = 1; for (int w = 0; w < B; w++) bd.pitems_max = std::max(bd.pitems_max, std::max(b->meta[w].npitems, b->meta[w].nmpitems));
    bd.pout_stride = bd.n_fused_wide ? (int)XL<true>::OUT : (int)XL<false>::OUT;
    bd.marg_nmax = b->prior_nmax;
    bd.env_max = 1; bd.nf_max = 1;
    for (int w = 0; w < B; w++) { bd.env_max = std::max(bd.env_max, b->meta[w].esize); bd.nf_max = std::max(bd.nf_max, b->meta[w].nf); }
    b->total_state = nstate;
    // ---- the slab: every array once -- its device field, its element count, and for an input its view in the staging slab (HostArrays).
    // Inputs come first and are uploaded as one block; a work array is never empty.
    struct Ent { void **dev, **host; size_t bytes, off; };
    std::vector<Ent> ents;
    HostArrays h; memset(&h, 0, sizeof h);
    auto IN = [&](auto **dev, auto *&host, size_t count) {
        static_assert(std::is_same<std::remove_const_t<std::remove_reference_t<decltype(**dev)>>, std::remove_reference_t<decltype(*host)>>::value, "host view of another type");
        ents.push_back({(void **)dev, (void **)&host, count * sizeof(*host), 0});
    };
    auto WK = [&](auto **dev, size_t count) { ents.push_back({(void **)dev, nullptr, (count ? count : 1) * sizeof(**dev), 0}); };
    IN(&bd.meta, h.meta, B); IN(&bd.prior, h.prior, npri); IN(&bd.vis_code, h.vis_code, nvis); IN(&bd.vis_lm, h.vis_lm, nvis); IN(&bd.vis_oi, h.vis_oi, nvis);
    if (!dev_obs) { IN(&bd.obs_i, h.obs_i, nobsi * 6); IN(&bd.obs_j, h.obs_j, nvis * 6); }
    IN(&bd.lm_win, h.lm_win, nlm); IN(&bd.lm_fptr, h.lm_fptr, nlm + 1);
    IN(&bd.items, h.items, nit_s + nit_m); IN(&bd.asm_list, h.asm_list, nlist);
    IN(&bd.imu_fi, h.imu_fi, nimu); IN(&bd.imu_fj, h.imu_fj, nimu); IN(&bd.imu_win, h.imu_win, nimu); IN(&bd.wheel_fi, h.wheel_fi, nwheel); IN(&bd.wheel_fj, h.wheel_fj, nwheel); IN(&bd.wheel_win, h.wheel_win, nwheel);
    IN(&bd.plane_f, h.plane_f, nplane); IN(&bd.plane_win, h.plane_win, nplane); IN(&bd.imu_data, h.imu_data, nimu * 287); IN(&bd.wheel_data, h.wheel_data, nwheel * 78);
    IN(&bd.prior_J, h.prior_J, npJ); IN(&bd.prior_r, h.prior_r, npr); IN(&bd.prior_x0, h.prior_x0, npri * SFIX); IN(&b->work_init_dev, h.work, B);
    if (dev_obs) { IN(&b->x_fix, h.x_fix, (size_t)B * SFIX); IN(&b->fm_off, h.fm_off, 2 * (size_t)B); } else IN(&bd.x_init, h.x_init, nstate);
    IN(&bd.vis_pos, h.vis_pos, bd.n_fused_wide ? nvis : 0); IN(&bd.lmb_desc, h.lmb_desc, nlmb); IN(&bd.pitems, h.pitems, npit);
    IN(&bd.mvis_pos, h.mvis_pos, nmpit ? nvis : 0); IN(&bd.mpitems, h.mpitems, nmpit);
    int *h_plan = nullptr; IN(&bd.chol_plan, h_plan, nplan);
    IN(&bd.run_desc, h.run_desc, nrun); IN(&bd.run_tile, h.run_tile, nrtile); IN(&bd.run_f, h.run_f, nrun ? nvis : 0); IN(&bd.run_lm, h.run_lm, nrun ? 2 * nlm : 0);
    const size_t nvec = (size_t)B * TFIX + nlm;
    const bool any_unfused = bd.n_unfused || bd.n_munfused;      // lin_vis' per-factor records and costs
    if (dev_obs) { WK(&bd.obs_i, nobsi * 6); WK(&bd.obs_j, nvis * 6); WK(&bd.x_init, nstate); }
    WK(&bd.work, B); WK(&bd.x_cur, nstate); WK(&bd.x_cand, nstate); WK(&bd.x_before, nstate);
    WK(&bd.vis_type, nvis); WK(&bd.vis_fi, nvis); WK(&bd.vis_fj, nvis); WK(&bd.vis_win, nvis); WK(&bd.vis_dup, nvis); WK(&bd.vis_obs, nvis * 12);
    WK(&bd.vis_rec, any_unfused ? nvis * VREC : 0); WK(&bd.vis_cost, any_unfused ? nvis : 0);
    WK(&bd.xrec, std::max(nxr, nmxr)); WK(&bd.pair_out, npit * (size_t)bd.pout_stride); WK(&bd.mpair_out, nmpit * (size_t)XL<true>::OUT); WK(&bd.pair_red, (npit || nmpit) ? (size_t)B * PAIR_RED : 0);
    WK(&bd.lm_a, nlm); WK(&bd.lm_g, nlm); WK(&bd.lm_gamma, nlm); WK(&bd.lm_scale, nlm); WK(&bd.lm_cost, nlm); WK(&bd.lm_W, nlm * VSUB); WK(&bd.lm_outlier, nlm);
    WK(&bd.imu_S, nimu * 225); WK(&bd.wheel_S, nwheel * 36); WK(&bd.imu_rec, nimu * IMU_REC); WK(&bd.wheel_rec, nwheel * WHEEL_REC); WK(&bd.plane_rec, nplane * PLANE_REC);
    WK(&bd.prior_A, npJ); WK(&bd.prior_res, npr); WK(&bd.prior_g, npr);
    WK(&bd.Hpk, (size_t)B * (TFIX * (TFIX + 1) / 2)); WK(&bd.gpk, (size_t)B * TFIX);
    WK(&bd.asm_out, (nit_s + nit_m) * ASM_STRIDE); WK(&bd.Tvis, (size_t)B * VSUB * VSUB); WK(&bd.tvec, (size_t)B * VSUB);
    WK(&bd.v_scale, nvec); WK(&bd.v_D, nvec); WK(&bd.v_sgrad, nvec); WK(&bd.v_gn, nvec); WK(&bd.v_wug, nlm); WK(&bd.v_wun, nlm);
    // marginalisation outputs / scratch: sized by the largest prior this batch produces, and not at all when no window marginalises
    const size_t mJ = b->any_marg ? (size_t)b->prior_nmax * b->prior_nmax : 0, mB = b->any_marg ? (size_t)B : 0;
    WK(&bd.marg_J, mB * mJ); WK(&bd.marg_r, mB * MAXPRI); WK(&bd.marg_x0, mB * SFIX);
    WK(&bd.marg_hdr, mB * (3 + 2 * NB)); WK(&bd.marg_de, mB * 2 * MAXPRI); WK(&bd.marg_rot, mB * 2 * marg_rot_cap(b->prior_nmax)); WK(&bd.marg_sweep, mB * (2 * marg_sweep_cap(b->prior_nmax) + 2));
    size_t tot = 0;
    for (auto &e : ents) if (e.host) { e.off = tot; tot += align_up(e.bytes); }
    const size_t in_bytes = tot;
    for (auto &e : ents) if (!e.host) { e.off = tot; tot += align_up(e.bytes); }
    b->out_bytes = align_up(nstate * 8) + align_up(sizeof(WinWork) * B) + align_up((size_t)B * (3 + 2 * NB) * 4) + align_up((size_t)B * MAXPRI * 8) +
                   align_up((size_t)B * SFIX * 8) + align_up((size_t)B * b->prior_nmax * b->prior_nmax * 8);
    b->out_off = align_up(in_bytes);
    const size_t host_need = b->out_off + b->out_bytes;
    Arena *ar;
    if (use_cached && !ctx->arena.busy) { ar = &ctx->arena; b->arena_cached = true; ctx->arena.busy = true; } else { ar = &b->arena; b->arena_cached = false; }
    if (ar->dev_cap < tot) { if (ar->dev) dev_free(ar->dev); ar->dev = nullptr; ar->dev_cap = 0; void *d = nullptr; int e = dev_malloc(&d, tot + tot / 8); if (e) { batch_free(ctx, b); return fail(ctx, VIWB_ERR_CUDA, std::string("device slab: ") + dev_errstr(e)); } ar->dev = (char *)d; ar->dev_cap = tot + tot / 8; }
    if (ar->host_cap < host_need) { if (ar->host) host_free(ar->host); ar->host = nullptr; ar->host_cap = 0; void *hm = nullptr; int e = host_alloc(&hm, host_need + host_need / 8); if (e) { batch_free(ctx, b); return fail(ctx, VIWB_ERR_CUDA, "pinned staging slab"); } ar->host = (char *)hm; ar->host_cap = host_need + host_need / 8; }
    if (b->arena_cached) b->arena = *ar;     // a view; ownership stays with the context
    const double t_alloc = now_ms();
    for (auto &e : ents) { *e.dev = ar->dev + e.off; if (e.host) *e.host = ar->host + e.off; }
    h.nitems_solve_total = (int)nit_s; h.meta_count = B;
    if (npri) memcpy(h.prior, priors.data(), sizeof(PriorDev) * npri);
    h.lm_fptr[nlm] = (int)nvis;
    for (const std::vector<int> &pl : plans) { memcpy(h_plan, pl.data(), sizeof(int) * pl.size()); h_plan += pl.size(); }
    // ---- phase 3 (parallel): fill
    std::vector<unsigned char> obs_viol(B, 0); h.obs_viol = obs_viol.data();
    parallel_for(B, [&](int w) { lower_fill(problems[w], states[w], w, b->meta[w], low[w], h, opt->initial_trust_region_radius); });
    if (!obs_per_factor && std::find(obs_viol.begin(), obs_viol.end(), 1) != obs_viol.end()) {      // rare: rebuild with one host-side entry per factor
        batch_free(ctx, b);
        return batch_build(ctx, B, problems, states, options, margin_flags, out, use_cached, true, from);
    }
    const double t_filled = now_ms();
    { int e = dev_h2d(ar->dev, ar->host, in_bytes, ctx->stream); if (e) { batch_free(ctx, b); return fail(ctx, VIWB_ERR_CUDA, std::string("H2D: ") + dev_errstr(e)); } }
    ctx->h2d_bytes += (long long)in_bytes;
    if (dev_obs) fm_fill_batch(from, b);
    if (nvis) LAUNCH(ctx, vis_expand, bd, B, 1, NT(128), 0, 0);      // code words + split observations -> the tables the kernels read
    { const int rc = launch_status(ctx); if (rc) { batch_free(ctx, b); return rc; } }
    // (no wait here: the kernels of the run are queued behind the upload on the same stream, the results are staged in their own region of the slab, and the
    //  slab is next written by the host only after a fetch has synchronised)
    if (g_timing) fprintf(stderr, "[viwb] build B=%d: plan+slabs %.2f ms (count %.2f), fill %.2f ms (%.1f MB), h2d %.2f ms\n", B, t_alloc - t_start, t_counted - t_start, t_filled - t_alloc, in_bytes / 1e6, now_ms() - t_filled);
    *out = b;
    return 0;
}

enum { RUN_SOLVE = 1, RUN_REANCHOR = 2, RUN_MARG = 4, RUN_LIN_ONLY = 8 };

// Threads per block of the batch's solve launch: SOLVE_NT, unless the widest window's shared memory leaves that kernel fewer resident warps per SM
// than the 384-thread one (both hold two such windows per SM, as for C4 windows): then SOLVE_WIDE_NT.  The emulation always runs solve_block.
static int solve_threads(const BatchDev &bd) {
#ifdef VIWB_HOST_EMU
    (void)bd;
    return SOLVE_NT;
#else
    int a = 0, b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, solve_kernel, SOLVE_NT, solve_smem_doubles(SOLVE_NT, bd.env_max, bd.nf_max) * 8) ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, solve_wide_kernel, SOLVE_WIDE_NT, solve_smem_doubles(SOLVE_WIDE_NT, bd.env_max, bd.nf_max) * 8))
        return SOLVE_NT;
    return a * SOLVE_NT >= b * SOLVE_WIDE_NT ? SOLVE_NT : SOLVE_WIDE_NT;
#endif
}
static int batch_execute(viwb_context *ctx, viwb_batch *b, int what) {
    bind_device(ctx);
    BatchDev &bd = b->bd;
    int rc = ensure_attrs(ctx); if (rc) return rc;
    stream_t st = ctx->stream;
    const int B = b->B;
    const size_t xs = b->total_state * sizeof(double);
    CK(dev_d2d(bd.x_cur, bd.x_init, xs, st)); CK(dev_d2d(bd.x_cand, bd.x_init, xs, st));
    if (!(what & RUN_REANCHOR) || (what & RUN_SOLVE)) CK(dev_d2d(bd.x_before, bd.x_init, xs, st));
    CK(dev_d2d(bd.work, b->work_init_dev, sizeof(WinWork) * B, st));
    const int nt_vis = NT(128), nt_lm = NT(128), nt_small = NT(128), nt_asm = NT(128), nt_solve = NT(SOLVE_NT), nt_marg = NT(256);
    const int g_vis = (bd.nvis_total + nt_vis - 1) / nt_vis, g_lm = (bd.nlm_total * LM_ROLES + nt_lm - 1) / nt_lm;
    const size_t sm_small = lin_small_smem_doubles(nt_small) * 8, sm_solve = solve_smem_doubles(nt_solve, bd.env_max, bd.nf_max) * 8, sm_marg = marg_prep_smem_doubles(nt_marg, bd.marg_nmax) * 8, sm_eig = marg_eig_smem_doubles(nt_marg, bd.marg_nmax) * 8;
    // cost_only: the round after the last allowed iteration only decides accept / reject of the pending candidate (every window
    // still running is at max_num_iterations there, trust_region_minimizer.cc checks the iteration limit before the gradient),
    // so the partial sums and the Schur product of that linearisation would never be read
    // one linearisation: visual kernels of the fused paths, then of the unfused windows, the small factors, (the accept / reject decision stops here),
    // the fused paths' pair products, the unfused windows' gather sums, and the Schur product
    auto lin = [&](int mode, bool cost_only) {
        const bool solve = mode == MODE_SOLVE;
        const bool unfused = solve ? bd.n_unfused > 0 : bd.n_munfused > 0;      // windows outside the fused path (irregular factor tables)
        const int vmode = cost_only ? (int)MODE_COST : mode;
        if (solve && bd.n_fused_compact > 0) LAUNCH(ctx, lin_vis_lm, bd, bd.nrun_total, 1, NT(LMB_FACTORS), lin_vis_run_smem_doubles() * 8, vmode);      // + the compact windows' pair chunks
        if (solve ? bd.n_fused_wide > 0 : bd.n_mfused > 0) LAUNCH(ctx, lin_vis_lm_wide, bd, bd.nlmb_total, 1, NT(LMB_FACTORS), lin_vis_lm_smem_doubles(true) * 8, vmode);
        if (unfused) {
            LAUNCH(ctx, lin_vis, bd, g_vis, 1, nt_vis, lin_vis_smem_doubles(nt_vis) * 8, mode);
            LAUNCH(ctx, lm_reduce, bd, g_lm, 1, nt_lm, 0, mode);
        }
        LAUNCH(ctx, lin_small, bd, B, 1, nt_small, sm_small, mode);
        if (cost_only) return;
        const int nfi = solve ? bd.npitems_total : bd.nmpitems_total, wpb = nt_asm / (nt_asm < 32 ? nt_asm : 32);
        if (nfi > 0) {
            if (!solve || bd.n_fused_wide > 0) LAUNCH(ctx, asm_pairs_wide, bd, (nfi + wpb - 1) / wpb, 1, NT(128), 0, mode);
            LAUNCH(ctx, pair_reduce, bd, B, 1, NT(PAIR_RED_NT), (size_t)bd.pitems_max * sizeof(int), mode);
        }
        if (unfused) LAUNCH(ctx, asm_items, bd, ((solve ? bd.nitems_solve : bd.nitems_marg) * ASM_SPLIT + wpb - 1) / wpb, 1, nt_asm, 0, mode);
        LAUNCH(ctx, syrk_mma, bd, B, 1, NT(SYRK_NT), syrk_mma_smem_doubles() * 8, mode);
    };
    if (what & (RUN_SOLVE | RUN_MARG | RUN_LIN_ONLY)) {
        const int ns = bd.nimu_total + bd.nwheel_total, nt_s = NT(128);
        LAUNCH(ctx, setup, bd, (ns + nt_s - 1) / nt_s, 1, nt_s, 0, 0);
        LAUNCH(ctx, prior_setup, bd, bd.nprior, 1, NT(256), 0, 0);
    }
    // the solve kernel at the block size that keeps more of its warps resident (solve_threads); both compute the same bits
    const int solve_nt = solve_threads(bd);
    const size_t sm_solve_at = solve_smem_doubles(solve_nt, bd.env_max, bd.nf_max) * 8;
    auto launch_solve = [&](int mode) {
        if (solve_nt == SOLVE_NT) LAUNCH(ctx, solve, bd, B, 1, nt_solve, sm_solve, mode);
        else KERNEL(ctx, "solve", B, 1, solve_nt, sm_solve_at, solve_wide_kernel, (bd, mode), emu_launch(solve_block, bd, B, 1, sm_solve_at, mode));
    };
    if (what & RUN_LIN_ONLY) { lin(MODE_SOLVE, false); launch_solve(2); }
    if (what & RUN_SOLVE) {
        // SOLVER_TIME (estimator.cpp:1650-1653): Ceres tests the wall clock after every iteration; here the host
        // waits for each round only when a limit is set, and the round after the limit just decides the pending
        // candidate and stops (NO_CONVERGENCE).  Disabled (0) keeps the whole solve asynchronous.
        const auto t_start = std::chrono::steady_clock::now();
        bool last = false;
        for (int round = 0; round <= b->max_iter && !last; round++) {
            if (b->max_time > 0.0 && round > 0) {
                CK(dev_sync(st));
                last = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() >= b->max_time;
            }
            lin(MODE_SOLVE, last || (round == b->max_iter && round > 0));
            launch_solve(last ? 3 : 0);
        }
    }
    if (what & RUN_REANCHOR) LAUNCH(ctx, reanchor, bd, B, 1, NT(32), 0, 0);
    if ((what & RUN_MARG) && b->any_marg) {
        lin(MODE_MARG, false);
        LAUNCH(ctx, marg_prep, bd, B, 1, nt_marg, sm_marg, 0);
        if (g_marg_one_kernel) LAUNCH(ctx, marg_eig, bd, B, 1, nt_marg, sm_eig, 0);
        else {
            LAUNCH(ctx, marg_tri, bd, B, 1, NT(MARG_TRI_NT), sm_eig, 0);
            LAUNCH(ctx, marg_ql, bd, B, 1, NT(32), 2 * MAXPRI * 8, 0);
            LAUNCH(ctx, marg_apply, bd, B, 1, NT(128), marg_apply_smem_doubles(128, bd.marg_nmax) * 8, 0);
        }
    }
    return launch_status(ctx);
}

static int batch_fetch(viwb_context *ctx, viwb_batch *b, double *const *states, viwb_summary *summaries, viwb_prior *priors_out) {
    bind_device(ctx);
    BatchDev &bd = b->bd;
    const int B = b->B, nmax = b->prior_nmax;
    // staging layout inside the pinned slab
    char *hs = b->arena.host + b->out_off;
    size_t o = 0;
    double *x = (double *)(hs + o); o += align_up(b->total_state * 8);
    WinWork *work = (WinWork *)(hs + o); o += align_up(sizeof(WinWork) * B);
    int *hdr = (int *)(hs + o); o += align_up((size_t)B * (3 + 2 * NB) * 4);
    double *r = (double *)(hs + o); o += align_up((size_t)B * MAXPRI * 8);
    double *x0 = (double *)(hs + o); o += align_up((size_t)B * SFIX * 8);
    double *J = (double *)(hs + o);
    CK(dev_d2h(x, bd.x_cur, b->total_state * sizeof(double), ctx->stream));
    CK(dev_d2h(work, bd.work, sizeof(WinWork) * B, ctx->stream));
    const bool want_pr = priors_out && b->any_marg;
    if (want_pr) {
        CK(dev_d2h(hdr, bd.marg_hdr, (size_t)B * (3 + 2 * NB) * sizeof(int), ctx->stream));
        CK(dev_d2h(r, bd.marg_r, (size_t)B * MAXPRI * sizeof(double), ctx->stream));
        CK(dev_d2h(x0, bd.marg_x0, (size_t)B * SFIX * sizeof(double), ctx->stream));
        CK(dev_d2h(J, bd.marg_J, (size_t)B * nmax * nmax * 8, ctx->stream));     // window w's n x n block (row stride n) heads its nmax^2 slot
    }
    CK(dev_sync(ctx->stream));
    std::atomic<int> marg_fail(0);
    parallel_for(B, [&](int w) {           // ~54 KB of prior per window: the unpack into the caller's buffers runs on the host pool
        if (states && states[w]) memcpy(states[w], x + b->meta[w].state_off, sizeof(double) * b->state_sizes[w]);
        if (summaries) {
            viwb_summary &sm = summaries[w]; const WinWork &ww = work[w];
            sm.termination_type = ww.term; sm.num_iterations = ww.num_iterations; sm.num_successful_steps = ww.successful; sm.num_linear_solves = ww.num_linear;
            sm.initial_cost = ww.initial_cost; sm.final_cost = ww.x_cost; sm.final_radius = ww.radius; sm.final_mu = ww.mu;
        }
        if (!priors_out) return;
        viwb_prior *out = &priors_out[w];
        const int mode = b->out_mode[w];
        if (mode == 0 && want_pr) {
            const int *h = hdr + (size_t)w * (3 + 2 * NB);
            out->valid = h[0]; out->n = h[1]; out->num_blocks = h[2];
            for (int i = 0; i < h[2]; i++) { out->block_id[i] = h[3 + i]; out->block_idx[i] = h[3 + NB + i]; }
            const int n = h[1];
            if (h[0]) {
                memcpy(out->J, J + (size_t)w * nmax * nmax, sizeof(double) * n * n);
                memcpy(out->r, r + (size_t)w * MAXPRI, sizeof(double) * n);
                memcpy(out->x0, x0 + (size_t)w * SFIX, sizeof(double) * SFIX);
            }
            if (work[w].marg_status < 0) marg_fail = work[w].marg_status;
        } else if (mode == 1) {
            const HostPrior &hp = b->in_prior[w];
            out->valid = 1; out->n = hp.n; out->num_blocks = hp.nb;
            memcpy(out->block_id, hp.block_id, sizeof hp.block_id); memcpy(out->block_idx, hp.block_idx, sizeof hp.block_idx);
            memcpy(out->x0, hp.x0.data(), sizeof(double) * SFIX); memcpy(out->J, hp.J.data(), sizeof(double) * hp.n * hp.n); memcpy(out->r, hp.r.data(), sizeof(double) * hp.n);
        } else { out->valid = 0; out->n = 0; out->num_blocks = 0; }
    });
    // marg_status: -1 from marg_prep (kept block larger than marg_cap), -2 from marg_ql (rotation or sweep log full)
    if (marg_fail == -1) return fail(ctx, VIWB_ERR_NUMERIC, "marginalisation: kept dimension exceeds the shared-memory eigen solver");
    if (marg_fail == -2) return fail(ctx, VIWB_ERR_NUMERIC, "marginalisation: the QL iteration filled its rotation log");
    if (marg_fail) return fail(ctx, VIWB_ERR_NUMERIC, "marginalisation failed");
    return 0;
}

static void batch_free(viwb_context *ctx, viwb_batch *b) {
    if (!b) return;
    if (ctx) dev_sync(ctx->stream);            // the upload of batch_build is not waited for there: nothing may still read the staging slab when it is released or reused
    if (b->arena_cached) { if (ctx) ctx->arena.busy = false; }
    else arena_release(b->arena);
    delete b;
}

// outliersRejection on the states the batch currently holds (after viwb_batch_run: the solved, re-anchored windows) -> bd.lm_outlier
static int batch_outlier_launch(viwb_context *ctx, viwb_batch *b, double focal_length, double threshold_px) {
    BatchDev bd = b->bd; bd.out_focal = focal_length; bd.out_thresh = threshold_px;
    const int nt = NT(128);
    LAUNCH(ctx, outlier, bd, (bd.nlm_total + nt - 1) / nt, 1, nt, 0, 0);
    return launch_status(ctx);
}

#include "features_batch.inl"

// ====================================================================================== C ABI
extern "C" int viwb_create(int device, viwb_context **out) {
    if (!out) return VIWB_ERR_INVALID;
    viwb_context *ctx = new viwb_context();
    ctx->device = device; ctx->launches = 0; ctx->h2d_bytes = 0; ctx->attrs_set = false; ctx->stream = 0; ctx->own_stream = 0; ctx->lk1 = nullptr; ctx->det1 = nullptr;
#ifndef VIWB_HOST_EMU
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || device < 0 || device >= count) { delete ctx; return VIWB_ERR_CUDA; }   // no CPU fallback: fail loudly
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return VIWB_ERR_CUDA; }
    if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return VIWB_ERR_CUDA; }
    ctx->stream = ctx->own_stream;
#endif
    *out = ctx;
    return VIWB_OK;
}
extern "C" void viwb_destroy(viwb_context *ctx) {
    if (!ctx) return;
    lk_batch_free(ctx->lk1);
    det_free(ctx->det1);
#ifndef VIWB_HOST_EMU
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
#endif
    arena_release(ctx->arena);
    delete ctx;
}
extern "C" const char *viwb_last_error(const viwb_context *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
// (NULL is CUDA's legacy default stream, a valid handle -- torch's current stream usually is it.)  Work already queued on the previous stream is
// waited for, so that buffers the context recycles (arena, staging slab) are never touched from two streams at once
extern "C" int viwb_set_stream(viwb_context *ctx, void *s) {
    if (!ctx) return VIWB_ERR_INVALID;
    bind_device(ctx);
    CK(dev_sync(ctx->stream));
    ctx->stream = (stream_t)s;
    return VIWB_OK;
}
extern "C" long long viwb_launch_count(const viwb_context *ctx) { return ctx ? ctx->launches : 0; }
extern "C" long long viwb_h2d_bytes(const viwb_context *ctx) { return ctx ? ctx->h2d_bytes : 0; }

extern "C" int viwb_set_profiling(viwb_context *ctx, int enable) {
    if (!ctx) return VIWB_ERR_INVALID;
#ifndef VIWB_HOST_EMU
    g_prof.collect(); g_prof.on = enable != 0;
    if (enable) { g_prof.names.clear(); g_prof.ms.clear(); g_prof.count.clear(); }
#else
    (void)enable;
#endif
    return VIWB_OK;
}
extern "C" int viwb_profile_count(viwb_context *ctx) {
    (void)ctx;
#ifndef VIWB_HOST_EMU
    g_prof.collect(); return (int)g_prof.names.size();
#else
    return 0;
#endif
}
extern "C" int viwb_profile_get(viwb_context *ctx, int idx, char *name, int name_cap, double *total_ms, long long *launches) {
    (void)ctx;
#ifndef VIWB_HOST_EMU
    if (idx < 0 || idx >= (int)g_prof.names.size()) return VIWB_ERR_INVALID;
    if (name && name_cap > 0) { strncpy(name, g_prof.names[idx].c_str(), name_cap - 1); name[name_cap - 1] = 0; }
    if (total_ms) *total_ms = g_prof.ms[idx];
    if (launches) *launches = g_prof.count[idx];
    return VIWB_OK;
#else
    (void)idx; (void)name; (void)name_cap; (void)total_ms; (void)launches; return VIWB_ERR_INVALID;
#endif
}

#if defined(VIWB_SOLVE_PROBE) && !defined(VIWB_HOST_EMU)
// phase probe of the solve kernel (libviwb_phases.so only; profiles/solve_phase_probe.py): per window, SPH_SLOTS counters --
// the cycles of each phase summed over the launches that computed a step, then the number of such launches and of factorisations
extern "C" int viwb_solve_probe_slots(void) { return SPH_SLOTS; }
extern "C" int viwb_solve_probe_clear(viwb_context *ctx) {
    bind_device(ctx);
    CK(cudaStreamSynchronize(ctx->stream));
    static const std::vector<unsigned long long> zero((size_t)SPH_MAXW * SPH_SLOTS, 0ull);
    CK(cudaMemcpyToSymbol(g_solve_phase, zero.data(), zero.size() * sizeof(unsigned long long)));
    return VIWB_OK;
}
extern "C" int viwb_solve_probe_read(viwb_context *ctx, int nwin, unsigned long long *out) {
    bind_device(ctx);
    if (nwin < 0 || nwin > SPH_MAXW) return fail(ctx, VIWB_ERR_INVALID, "viwb_solve_probe_read: nwin out of range");
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaMemcpyFromSymbol(out, g_solve_phase, (size_t)nwin * SPH_SLOTS * sizeof(unsigned long long)));
    return VIWB_OK;
}
#endif

extern "C" int viwb_batch_create(viwb_context *ctx, int batch, const viwb_problem *problems, const double *const *states,
                                 const viwb_options *options, const int32_t *margin_flags, viwb_batch **out) {
    if (!ctx || !out) return VIWB_ERR_INVALID;
    int rc = batch_build(ctx, batch, problems, states, options, margin_flags, out);
    if (rc) return rc;
    CK(dev_sync(ctx->stream));
    return VIWB_OK;
}
// the windows as uploaded: current and candidate states back to the initial ones, solver bookkeeping cleared (viwb_batch_run does the same before it starts;
// this entry lets a caller read / evaluate the pristine batch, e.g. viwb_batch_outliers on the initial guess)
extern "C" int viwb_batch_reset_states(viwb_context *ctx, viwb_batch *b) {
    if (!ctx || !b) return VIWB_ERR_INVALID;
    bind_device(ctx);
    const size_t xs = b->total_state * sizeof(double);
    CK(dev_d2d(b->bd.x_cur, b->bd.x_init, xs, ctx->stream)); CK(dev_d2d(b->bd.x_cand, b->bd.x_init, xs, ctx->stream)); CK(dev_d2d(b->bd.x_before, b->bd.x_init, xs, ctx->stream));
    CK(dev_d2d(b->bd.work, b->work_init_dev, sizeof(WinWork) * b->B, ctx->stream));
    return VIWB_OK;
}
extern "C" int viwb_batch_run(viwb_context *ctx, viwb_batch *b) {
    if (!ctx || !b) return VIWB_ERR_INVALID;
    return batch_execute(ctx, b, RUN_SOLVE | RUN_REANCHOR | RUN_MARG);
}
extern "C" int viwb_batch_download(viwb_context *ctx, viwb_batch *b, double *const *states, viwb_summary *summaries, viwb_prior *priors_out) {
    if (!ctx || !b) return VIWB_ERR_INVALID;
    return batch_fetch(ctx, b, states, summaries, priors_out);
}
// outliersRejection on the states the batch currently holds, verdicts to the host
extern "C" int viwb_batch_outliers(viwb_context *ctx, viwb_batch *b, double focal_length, double threshold_px, uint8_t *const *outliers) {
    if (!ctx || !b || !outliers) return VIWB_ERR_INVALID;
    bind_device(ctx);
    const BatchDev &bd = b->bd;
    const int rc = batch_outlier_launch(ctx, b, focal_length, threshold_px); if (rc) return rc;
    std::vector<int> h(bd.nlm_total > 0 ? bd.nlm_total : 1);
    CK(dev_d2h(h.data(), bd.lm_outlier, (size_t)bd.nlm_total * sizeof(int), ctx->stream));
    CK(dev_sync(ctx->stream));
    for (int w = 0; w < b->B; w++) if (outliers[w]) { const WinMeta &m = b->meta[w]; for (int k = 0; k < m.nlm; k++) outliers[w][k] = (uint8_t)h[m.lm_off + k]; }
    return VIWB_OK;
}
extern "C" double viwb_batch_algorithmic_bytes(const viwb_batch *b) { return b ? b->algorithmic_bytes : 0.0; }
extern "C" int viwb_batch_solve_launch(viwb_context *ctx, const viwb_batch *b, int *threads, int *smem_bytes, int *blocks_per_sm) {
    if (!ctx || !b) return fail(ctx, VIWB_ERR_INVALID, "viwb_batch_solve_launch: null argument");
    bind_device(ctx);
    int rc = ensure_attrs(ctx); if (rc) return rc;
    const int nt = solve_threads(b->bd), smem = (int)(solve_smem_doubles(nt, b->bd.env_max, b->bd.nf_max) * 8);
    if (threads) *threads = nt;
    if (smem_bytes) *smem_bytes = smem;
    if (blocks_per_sm) {
#ifdef VIWB_HOST_EMU
        return fail(ctx, VIWB_ERR_INVALID, "viwb_batch_solve_launch: no device in the emulation");
#else
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, nt == SOLVE_NT ? (const void *)solve_kernel : (const void *)solve_wide_kernel, nt, (size_t)smem));
#endif
    }
    return VIWB_OK;
}
extern "C" void viwb_batch_destroy(viwb_context *ctx, viwb_batch *b) { batch_free(ctx, b); }

static int run_once(viwb_context *ctx, int B, const viwb_problem *problems, double *const *states, const viwb_options *opt,
                    const int32_t *flags, int what, viwb_summary *summaries, viwb_prior *priors, const double *const *before) {
    viwb_batch *b = nullptr;
    int rc = batch_build(ctx, B, problems, (const double *const *)states, opt, flags, &b, true);
    if (rc) return rc;
    if (before) {   // gauge re-anchoring against an explicit pre-solve state
        std::vector<double> xb(b->total_state);
        for (int w = 0; w < B; w++) memcpy(xb.data() + b->meta[w].state_off, before[w], sizeof(double) * b->state_sizes[w]);
        rc = dev_h2d(b->bd.x_before, xb.data(), xb.size() * sizeof(double), ctx->stream);
        if (!rc) rc = dev_sync(ctx->stream);
        if (rc) { batch_free(ctx, b); return fail(ctx, VIWB_ERR_CUDA, "upload of state_before failed"); }
    }
    const double t0 = now_ms();
    rc = batch_execute(ctx, b, what);
    if (g_timing) { dev_sync(ctx->stream); fprintf(stderr, "[viwb] execute %.2f ms\n", now_ms() - t0); }
    const double t1 = now_ms();
    if (!rc) rc = batch_fetch(ctx, b, states, summaries, priors);
    if (g_timing) fprintf(stderr, "[viwb] fetch %.2f ms\n", now_ms() - t1);
    batch_free(ctx, b);
    return rc;
}

extern "C" int viwb_window_solve(viwb_context *ctx, const viwb_problem *problem, double *state, const viwb_options *options, viwb_summary *summary) {
    if (!ctx || !problem || !state) return VIWB_ERR_INVALID;
    double *sp[1] = {state};
    return run_once(ctx, 1, problem, sp, options, nullptr, RUN_SOLVE, summary, nullptr, nullptr);
}
extern "C" int viwb_gauge_reanchor(viwb_context *ctx, const viwb_problem *problem, const double *state_before, double *state) {
    if (!ctx || !problem || !state || !state_before) return VIWB_ERR_INVALID;
    double *sp[1] = {state}; const double *bp[1] = {state_before};
    return run_once(ctx, 1, problem, sp, nullptr, nullptr, RUN_REANCHOR, nullptr, nullptr, bp);
}
extern "C" int viwb_outlier_rejection(viwb_context *ctx, const viwb_problem *problem, const double *state, double focal_length, double threshold_px,
                                      uint8_t *outliers) {
    if (!ctx || !problem || !state || !outliers) return VIWB_ERR_INVALID;
    viwb_batch *b = nullptr;
    const double *sp[1] = {state};
    int rc = batch_build(ctx, 1, problem, sp, nullptr, nullptr, &b, true);
    if (rc) return rc;
    rc = batch_execute(ctx, b, 0);                     // x_cur <- the given state, nothing else
    uint8_t *op[1] = {outliers};
    if (!rc) rc = viwb_batch_outliers(ctx, b, focal_length, threshold_px, op);
    batch_free(ctx, b);
    return rc;
}
extern "C" int viwb_marginalize(viwb_context *ctx, const viwb_problem *problem, const double *state, int margin_flag, viwb_prior *prior_out) {
    if (!ctx || !problem || !state || !prior_out) return VIWB_ERR_INVALID;
    std::vector<double> tmp(state, state + SFIX + problem->num_landmarks);
    double *sp[1] = {tmp.data()}; int32_t fl[1] = {margin_flag};
    return run_once(ctx, 1, problem, sp, nullptr, fl, RUN_MARG, nullptr, prior_out, nullptr);
}
extern "C" int viwb_optimization(viwb_context *ctx, const viwb_problem *problem, double *state, const viwb_options *options, int margin_flag,
                                 viwb_summary *summary, viwb_prior *prior_out) {
    if (!ctx || !problem || !state) return VIWB_ERR_INVALID;
    double *sp[1] = {state}; int32_t fl[1] = {margin_flag};
    return run_once(ctx, 1, problem, sp, options, prior_out ? fl : nullptr, RUN_SOLVE | RUN_REANCHOR | (prior_out ? RUN_MARG : 0), summary, prior_out, nullptr);
}
extern "C" int viwb_optimization_batch(viwb_context *ctx, int batch, const viwb_problem *problems, double *const *states, const viwb_options *options,
                                       const int32_t *margin_flags, viwb_summary *summaries, viwb_prior *priors_out) {
    if (!ctx || !problems || !states) return VIWB_ERR_INVALID;
    return run_once(ctx, batch, problems, states, options, priors_out ? margin_flags : nullptr, RUN_SOLVE | RUN_REANCHOR | (priors_out ? RUN_MARG : 0),
                    summaries, priors_out, nullptr);
}

extern "C" int viwb_debug_normal_equations(viwb_context *ctx, const viwb_problem *problem, const double *state, double *H, double *g, double *lm, double *cost) {
    if (!ctx || !problem || !state) return VIWB_ERR_INVALID;
    viwb_batch *b = nullptr;
    const double *sp[1] = {state};
    int rc = batch_build(ctx, 1, problem, sp, nullptr, nullptr, &b);
    if (rc) return rc;
    rc = batch_execute(ctx, b, RUN_LIN_ONLY);
    if (rc) { batch_free(ctx, b); return rc; }
    const int N = problem->num_landmarks;
    std::vector<double> Hd((size_t)TFIX * (TFIX + 1) / 2), gd(TFIX), a(N + 1), gl(N + 1), W((size_t)(N + 1) * VSUB), lc(N + 1);
    std::vector<WinWork> ww(1);
    int e = dev_d2h(Hd.data(), b->bd.Hpk, Hd.size() * 8, ctx->stream);
    e |= dev_d2h(gd.data(), b->bd.gpk, gd.size() * 8, ctx->stream);
    e |= dev_d2h(a.data(), b->bd.lm_a, (size_t)N * 8, ctx->stream); e |= dev_d2h(gl.data(), b->bd.lm_g, (size_t)N * 8, ctx->stream);
    e |= dev_d2h(W.data(), b->bd.lm_W, (size_t)N * VSUB * 8, ctx->stream); e |= dev_d2h(lc.data(), b->bd.lm_cost, (size_t)N * 8, ctx->stream);
    e |= dev_d2h(ww.data(), b->bd.work, sizeof(WinWork), ctx->stream);
    e |= dev_sync(ctx->stream);
    if (e) { batch_free(ctx, b); return fail(ctx, VIWB_ERR_CUDA, "download failed"); }
    // formatting only: scatter the packed active triangle into the caller's fixed-layout arrays
    const WinMeta &m = b->meta[0];
    if (H) { memset(H, 0, sizeof(double) * TFIX * TFIX);
        std::vector<int> rp(m.nf + 1, 0);
        for (int i = 0; i < m.nf; i++) rp[i + 1] = rp[i] + i - m.efirst[i] + 1;      // skyline row pointers
        for (int ba = 0; ba < NB; ba++) for (int bb = 0; bb < NB; bb++) if (m.tcol[ba] >= 0 && m.tcol[bb] >= 0)
            for (int p = 0; p < blk_tsize(ba); p++) for (int q = 0; q < blk_tsize(bb); q++) {
                int ci = m.tcol[ba] + p, cj = m.tcol[bb] + q;
                if (ci < cj) std::swap(ci, cj);
                H[(blk_toff(ba) + p) * TFIX + blk_toff(bb) + q] = cj >= m.efirst[ci] ? Hd[(size_t)rp[ci] - m.efirst[ci] + cj] : 0.0;   // outside the envelope: structural zero
            } }
    if (g) { memset(g, 0, sizeof(double) * TFIX); for (int ba = 0; ba < NB; ba++) if (m.tcol[ba] >= 0) for (int p = 0; p < blk_tsize(ba); p++) g[blk_toff(ba) + p] = gd[m.tcol[ba] + p]; }
    double c = ww[0].small_cost;
    for (int k = 0; k < N; k++) {
        c += lc[k];
        if (lm) { lm[k * 82] = a[k]; lm[k * 82 + 1] = gl[k];
            for (int p = 0; p < VSUB; p++) {
                bool act = true;
                if (p < 66) act = m.tcol[p / 6] >= 0; else if (p < 72) act = m.tcol[BLK_EX0] >= 0; else if (p < 78) act = m.tcol[BLK_EX1] >= 0; else if (p == 78) act = m.tcol[BLK_TD] >= 0; else act = false;
                lm[k * 82 + 2 + p] = act ? W[(size_t)k * VSUB + p] : 0.0;
            } }
    }
    if (cost) *cost = c;
    batch_free(ctx, b);
    return VIWB_OK;
}

// -------------------------------------------------------------------------------------- factor level
struct EvalArgs { int type, want_j; const double *in; double *out; };
// in : globals(11) | consts(287) | params(7 blocks x 9)        out: residual(15) | tangent Jacobian (15 x 30)
VIWB_D void eval_factor_device(const EvalArgs &a) {
    const double *gl = a.in, *c = a.in + 11, *p = a.in + 11 + 287;
    double *r = a.out, *J = a.out + 15;
    const double *P[7]; for (int i = 0; i < 7; i++) P[i] = p + 9 * i;
    if (a.type <= 2) {
        VisOut o;
        if (a.type == 0) vis_eval(0, c, P[0], P[1], P[2], P[2], P[3][0], P[4][0], gl + 3, a.want_j != 0, o);
        else if (a.type == 1) vis_eval(1, c, P[0], P[1], P[2], P[3], P[4][0], P[5][0], gl + 3, a.want_j != 0, o);
        else vis_eval(2, c, P[0], P[0], P[0], P[1], P[2][0], P[3][0], gl + 3, a.want_j != 0, o);
        r[0] = o.r[0]; r[1] = o.r[1];
        if (a.want_j) { for (int k = 0; k < 12; k++) { J[k] = o.JA[k]; J[12 + k] = o.JB[k]; J[24 + k] = o.JE0[k]; J[36 + k] = o.JE1[k]; } J[48] = o.Jl[0]; J[49] = o.Jl[1]; J[50] = o.Jtd[0]; J[51] = o.Jtd[1]; }
    } else if (a.type == 3) {
        double S[225]; sqrt_info_upper(15, c + 62, S);
        imu_eval(c, S, gl, P[0], P[1], P[2], P[3], a.want_j != 0, r, J);
    } else if (a.type == 4) {
        double S[36]; sqrt_info_upper(6, c + 25, S);
        wheel_eval(c, S, P[0], P[1], P[2], P[3][0], P[4][0], P[5][0], P[6][0], a.want_j != 0, r, J);
    } else {
        plane_eval(gl + 7, P[0], P[1], P[2], P[3][0], a.want_j != 0, r, J);
    }
}
#ifndef VIWB_HOST_EMU
__global__ void eval_factor_kernel(EvalArgs a) { if (threadIdx.x == 0 && blockIdx.x == 0) eval_factor_device(a); }
#endif

extern "C" int viwb_factor_evaluate(viwb_context *ctx, int type, const viwb_globals *gl, const double *consts, const double *const *params,
                                    double *residuals, double **jacobians) {
    if (!ctx || !gl || !params || !residuals || type < 0 || type > 5) return VIWB_ERR_INVALID;
    static const int nblk[6] = {5, 6, 4, 4, 7, 4};
    static const int sizes[6][7] = {{7, 7, 7, 1, 1, 0, 0}, {7, 7, 7, 7, 1, 1, 0}, {7, 7, 1, 1, 0, 0, 0}, {7, 9, 7, 9, 0, 0, 0}, {7, 7, 7, 1, 1, 1, 1}, {7, 7, 4, 1, 0, 0, 0}};
    static const int nres[6] = {2, 2, 2, 15, 6, 3};
    static const int ncons[6] = {12, 12, 12, 287, 78, 0};
    std::vector<double> in(11 + 287 + 63, 0.0), out(15 + 450, 0.0);
    for (int k = 0; k < 3; k++) in[k] = gl->G[k];
    for (int k = 0; k < 4; k++) in[3 + k] = gl->vis_sqrt_info[k];
    for (int k = 0; k < 3; k++) in[7 + k] = gl->plane_sqrt_info[k];
    in[10] = gl->huber_delta;
    if (ncons[type]) { if (!consts) return VIWB_ERR_INVALID; memcpy(in.data() + 11, consts, sizeof(double) * ncons[type]); }
    for (int i = 0; i < nblk[type]; i++) memcpy(in.data() + 11 + 287 + 9 * i, params[i], sizeof(double) * sizes[type][i]);
    EvalArgs a; a.type = type; a.want_j = jacobians ? 1 : 0;
    const int rc = staged(ctx, "factor_evaluate", {stage_in(a.in, in.data(), in.size() * 8), stage_out(a.out, out.data(), out.size() * 8)}, [&] {
        KERNEL(ctx, "eval_factor", 1, 1, 32, 0, eval_factor_kernel, (a), eval_factor_device(a));
    });
    if (rc) return rc;
    for (int i = 0; i < nres[type]; i++) residuals[i] = out[i];
    if (jacobians) {   // formatting only: tangent columns -> the reference's row-major (rows x global size) blocks, last pose column zero
        const double *J = out.data() + 15;
        int ld = 0, tcol[7];
        if (type <= 2) {   // record layout A | B | E0 | E1 | l | td, 2 rows each
            const int off0[5] = {0, 12, 24, 48, 50}, off1[6] = {0, 12, 24, 36, 48, 50}, off2[4] = {24, 36, 48, 50};
            const int *off = type == 0 ? off0 : type == 1 ? off1 : off2;
            for (int i = 0; i < nblk[type]; i++) {
                if (!jacobians[i]) continue;
                const int gs = sizes[type][i], ts = gs == 7 ? 6 : 1;
                for (int r = 0; r < 2; r++) { for (int c2 = 0; c2 < ts; c2++) jacobians[i][r * gs + c2] = J[off[i] + r * ts + c2]; if (gs == 7) jacobians[i][r * gs + 6] = 0.0; }
            }
        } else {
            int c0 = 0;
            for (int i = 0; i < nblk[type]; i++) { tcol[i] = c0; const int gs = sizes[type][i]; c0 += gs == 7 ? 6 : gs == 4 ? 3 : gs; }
            ld = c0;
            for (int i = 0; i < nblk[type]; i++) {
                if (!jacobians[i]) continue;
                const int gs = sizes[type][i], ts = gs == 7 ? 6 : gs == 4 ? 3 : gs;
                for (int r = 0; r < nres[type]; r++) { for (int c2 = 0; c2 < ts; c2++) jacobians[i][r * gs + c2] = J[r * ld + tcol[i] + c2]; for (int c2 = ts; c2 < gs; c2++) jacobians[i][r * gs + c2] = 0.0; }
            }
        }
    }
    return VIWB_OK;
}

struct PriorEvalArgs { PriorDev p; const double *J, *r, *x0, *x; double *res; };
VIWB_D void prior_eval_device(const PriorEvalArgs &a, int tid, int nt, double *dx) {
    if (tid == 0) prior_dx(a.p, a.x, a.x0, dx);
    VIWB_SYNC();
    for (int i = tid; i < a.p.n; i += nt) { double s = a.r[i]; for (int k = 0; k < a.p.n; k++) s += a.J[i * a.p.n + k] * dx[k]; a.res[i] = s; }
}
#ifndef VIWB_HOST_EMU
__global__ void prior_eval_kernel(PriorEvalArgs a) { __shared__ double dx[MAXPRI]; prior_eval_device(a, threadIdx.x, blockDim.x, dx); }
#endif
extern "C" int viwb_prior_evaluate(viwb_context *ctx, const viwb_prior *prior, const double *state, double *residuals, double *jacobian) {
    if (!ctx || !prior || !state || !residuals || prior->n <= 0 || prior->n > MAXPRI) return VIWB_ERR_INVALID;
    const int n = prior->n;
    PriorEvalArgs a; memset(&a, 0, sizeof a);
    a.p.n = n; a.p.nb = prior->num_blocks;
    for (int i = 0; i < prior->num_blocks; i++) { a.p.block_id[i] = prior->block_id[i]; a.p.block_idx[i] = prior->block_idx[i]; }
    const int rc = staged(ctx, "prior_evaluate", {stage_in(a.J, prior->J, (size_t)n * n * 8), stage_in(a.r, prior->r, (size_t)n * 8), stage_in(a.x0, prior->x0, SFIX * 8),
                                                  stage_in(a.x, state, SFIX * 8), stage_out(a.res, residuals, (size_t)n * 8)}, [&] {
        KERNEL(ctx, "prior_eval", 1, 1, 128, 0, prior_eval_kernel, (a), double dx[MAXPRI]; prior_eval_device(a, 0, 1, dx));
    });
    if (rc) return rc;
    if (jacobian) {   // formatting only (marginalization_factor.cpp:381-394): J_lin columns at the block's state offset
        memset(jacobian, 0, sizeof(double) * n * SFIX);
        for (int i = 0; i < prior->num_blocks; i++) {
            const int bq = prior->block_id[i], ls = blk_msize(bq), idx = prior->block_idx[i], off = blk_off(bq);
            for (int r = 0; r < n; r++) for (int k = 0; k < ls; k++) jacobian[(size_t)r * SFIX + off + k] = prior->J[(size_t)r * n + idx + k];
        }
    }
    return VIWB_OK;
}

// -------------------------------------------------------------------------------------- pre-integration (SURVEY 8 f-2)
// interval i owns counts[i] steps of dt and counts[i] + 1 rows of samples; off: the first step of every interval
static int preint_offsets(viwb_context *ctx, int n, const int32_t *counts, std::vector<int> &off) {
    off.assign(n + 1, 0);
    for (int i = 0; i < n; i++) { if (counts[i] < 0) return fail(ctx, VIWB_ERR_INVALID, "negative sample count"); off[i + 1] = off[i] + counts[i]; }
    return VIWB_OK;
}

extern "C" int viwb_imu_preintegrate(viwb_context *ctx, int n, const int32_t *counts, const double *dt, const double *acc, const double *gyr,
                                     const double *ba, const double *bg, const double *noise, double *records) {
    if (!ctx || n < 0 || !counts || !dt || !acc || !gyr || !ba || !bg || !noise || !records) return VIWB_ERR_INVALID;
    if (n == 0) return VIWB_OK;
    std::vector<int> off; const int rc = preint_offsets(ctx, n, counts, off); if (rc) return rc;
    const size_t steps = off[n], rows = steps + n;
    ImuPreArgs a; a.n = n; for (int k = 0; k < 4; k++) a.noise[k] = noise[k];
    return staged(ctx, "imu_preintegrate", {stage_in(a.off, off.data(), off.size() * 4), stage_in(a.dt, dt, steps * 8), stage_in(a.acc, acc, rows * 24), stage_in(a.gyr, gyr, rows * 24),
                                            stage_in(a.ba, ba, (size_t)n * 24), stage_in(a.bg, bg, (size_t)n * 24), stage_out(a.rec, records, (size_t)n * 287 * 8)}, [&] {
        KERNEL(ctx, "imu_preint", (n + PRE_WPB - 1) / PRE_WPB, 1, 32 * PRE_WPB, PRE_WPB * PRE_IMU_SMEM * 8, imu_preint_kernel, (a),
               std::vector<double> sm(PRE_IMU_SMEM); for (int i = 0; i < n; i++) imu_preint_warp(a, i, 0, 1, sm.data()));
    });
}
extern "C" int viwb_wheel_preintegrate(viwb_context *ctx, int n, const int32_t *counts, const double *dt, const double *vel, const double *gyr,
                                       const double *s, const double *td, const double *noise, double *records) {
    if (!ctx || n < 0 || !counts || !dt || !vel || !gyr || !s || !td || !noise || !records) return VIWB_ERR_INVALID;
    if (n == 0) return VIWB_OK;
    std::vector<int> off; const int rc = preint_offsets(ctx, n, counts, off); if (rc) return rc;
    const size_t steps = off[n], rows = steps + n;
    WheelPreArgs a; a.n = n; a.noise[0] = noise[0]; a.noise[1] = noise[1];
    return staged(ctx, "wheel_preintegrate", {stage_in(a.off, off.data(), off.size() * 4), stage_in(a.dt, dt, steps * 8), stage_in(a.vel, vel, rows * 24), stage_in(a.gyr, gyr, rows * 24),
                                              stage_in(a.s, s, (size_t)n * 24), stage_in(a.td, td, (size_t)n * 8), stage_out(a.rec, records, (size_t)n * 78 * 8)}, [&] {
        KERNEL(ctx, "wheel_preint", (n + PRE_WPB - 1) / PRE_WPB, 1, 32 * PRE_WPB, PRE_WPB * PRE_WHEEL_SMEM * 8, wheel_preint_kernel, (a),
               std::vector<double> sm(PRE_WHEEL_SMEM); for (int i = 0; i < n; i++) wheel_preint_warp(a, i, 0, 1, sm.data()));
    });
}

// -------------------------------------------------------------------------------------- initialisation alignment (SURVEY 8 f-4 ii)
// the normal equations of both solves: A (two n x n matrices: linear alignment factors a copy), b, x, the pivots; n = 3 F + 4
extern "C" int viwb_solve_gyroscope_bias(viwb_context *ctx, int num_frames, const double *R, const double *imu_data, double *delta_bg) {
    if (!ctx || !R || !imu_data || !delta_bg) return VIWB_ERR_INVALID;
    if (num_frames < 2 || num_frames > VIWB_MAX_INIT_FRAMES) return fail(ctx, VIWB_ERR_INVALID, "solve_gyroscope_bias: 2..VIWB_MAX_INIT_FRAMES frames");
    const int F = num_frames, n = 3 * F + 4;
    GyroBiasArgs a; a.F = F;
    return staged(ctx, "solve_gyroscope_bias", {stage_in(a.R, R, (size_t)F * 72), stage_in(a.imu, imu_data, (size_t)(F - 1) * VIWB_IMU_DOUBLES * 8), stage_tmp(a.A, (size_t)2 * n * n * 8),
                                                stage_tmp(a.b, (size_t)(n + 8) * 8), stage_tmp(a.x, (size_t)(n + 8) * 8), stage_tmp(a.perm, (size_t)n * 4), stage_out(a.out, delta_bg, 24)}, [&] {
        KERNEL(ctx, "gyro_bias", 1, 1, 32, 0, gyro_bias_kernel, (a), gyro_bias_block(a, 0, 1));
    });
}

extern "C" int viwb_linear_alignment(viwb_context *ctx, int num_frames, const double *R, const double *T, const double *imu_data, const double *wheel_data,
                                     const double *tic, const double *rio, const double *tio, double g_norm, double *g, double *x, int32_t *x_size, int32_t *aligned) {
    if (!ctx || !R || !T || !imu_data || !tic || !g || !x || !x_size || !aligned || (wheel_data && (!rio || !tio))) return VIWB_ERR_INVALID;
    if (num_frames < 2 || num_frames > VIWB_MAX_INIT_FRAMES) return fail(ctx, VIWB_ERR_INVALID, "linear_alignment: 2..VIWB_MAX_INIT_FRAMES frames");
    const int F = num_frames, n = 3 * F + 4;
    std::vector<double> out((size_t)n + 5);
    AlignArgs a; a.F = F; a.use_wheel = wheel_data ? 1 : 0;
    memcpy(a.tic, tic, 24); a.g_norm = g_norm;
    for (int k = 0; k < 9; k++) a.rio[k] = rio ? rio[k] : (k % 4 == 0 ? 1.0 : 0.0);
    for (int k = 0; k < 3; k++) a.tio[k] = tio ? tio[k] : 0.0;
    const int rc = staged(ctx, "linear_alignment", {stage_in(a.R, R, (size_t)F * 72), stage_in(a.T, T, (size_t)F * 24), stage_in(a.imu, imu_data, (size_t)(F - 1) * VIWB_IMU_DOUBLES * 8),
                                                    stage_in(a.wheel, wheel_data, (size_t)(F - 1) * VIWB_WHEEL_DOUBLES * 8), stage_tmp(a.A, (size_t)2 * n * n * 8), stage_tmp(a.b, (size_t)(n + 8) * 8),
                                                    stage_tmp(a.x, (size_t)(n + 8) * 8), stage_tmp(a.perm, (size_t)n * 4), stage_out(a.out, out.data(), out.size() * 8)}, [&] {
        KERNEL(ctx, "align", 1, 1, 128, 0, align_kernel, (a), align_block(a, 0, 1));
    });
    if (rc) return rc;
    *aligned = out[0] != 0.0; memcpy(g, out.data() + 1, 24); *x_size = (int32_t)out[4];
    memcpy(x, out.data() + 5, (size_t)*x_size * 8);
    return VIWB_OK;
}

// -------------------------------------------------------------------------------------- triangulation / depth shift (SURVEY 8 f-3)
extern "C" int viwb_triangulate(viwb_context *ctx, const double *state, int n, const int32_t *stereo, const int32_t *frame, const double *pt0, const double *pt1,
                                double init_depth, double *depth) {
    if (!ctx || !state || n < 0 || !stereo || !frame || !pt0 || !pt1 || !depth) return VIWB_ERR_INVALID;
    if (n == 0) return VIWB_OK;
    for (int k = 0; k < n; k++) if (frame[k] < 0 || frame[k] + (stereo[k] ? 0 : 1) > VIWB_WINDOW_SIZE) return fail(ctx, VIWB_ERR_INVALID, "triangulate: frame index out of the window");
    TriArgs a; a.n = n; a.init_depth = init_depth;
    return staged(ctx, "triangulate", {stage_in(a.state, state, SFIX * 8), stage_in(a.stereo, stereo, (size_t)n * 4), stage_in(a.frame, frame, (size_t)n * 4),
                                       stage_in(a.pt0, pt0, (size_t)n * 16), stage_in(a.pt1, pt1, (size_t)n * 16), stage_out(a.depth, depth, (size_t)n * 8)}, [&] {
        KERNEL(ctx, "triangulate", (n + 127) / 128, 1, 128, 0, triangulate_kernel, (a), for (int k = 0; k < n; k++) triangulate_item(a, k));
    });
}
extern "C" int viwb_shift_depth(viwb_context *ctx, int n, const double *uv, const double *depth_in, const double *marg_R, const double *marg_P,
                                const double *new_R, const double *new_P, double init_depth, double *depth_out) {
    if (!ctx || n < 0 || !uv || !depth_in || !marg_R || !marg_P || !new_R || !new_P || !depth_out) return VIWB_ERR_INVALID;
    if (n == 0) return VIWB_OK;
    ShiftArgs a; a.n = n; a.init_depth = init_depth;
    memcpy(a.margR, marg_R, 72); memcpy(a.margP, marg_P, 24); memcpy(a.newR, new_R, 72); memcpy(a.newP, new_P, 24);
    return staged(ctx, "shift_depth", {stage_in(a.uv, uv, (size_t)n * 24), stage_in(a.depth_in, depth_in, (size_t)n * 8), stage_out(a.depth_out, depth_out, (size_t)n * 8)}, [&] {
        KERNEL(ctx, "shift_depth", (n + 127) / 128, 1, 128, 0, shift_depth_kernel, (a), for (int k = 0; k < n; k++) shift_depth_item(a, k));
    });
}
// Estimator::predictPtsInNextFrame (estimator.cpp:2080-2113): thread per feature of the caller's FeatureManager::feature list
extern "C" int viwb_predict_pts(viwb_context *ctx, const double *state, int frame_count, int n, const int32_t *start_frame, const int32_t *num_obs, const double *pt0,
                                const double *depth, double *pts_cam, uint8_t *valid) {
    if (!ctx || !state || n < 0 || !start_frame || !num_obs || !pt0 || !depth || !pts_cam || !valid) return VIWB_ERR_INVALID;
    if (frame_count < 0 || frame_count > VIWB_WINDOW_SIZE) return fail(ctx, VIWB_ERR_INVALID, "predict_pts: frame_count out of the window");
    for (int k = 0; k < n; k++) if (start_frame[k] < 0 || start_frame[k] > VIWB_WINDOW_SIZE || num_obs[k] < 0) return fail(ctx, VIWB_ERR_INVALID, "predict_pts: start_frame out of the window or negative num_obs");
    if (n == 0) return VIWB_OK;
    PredictArgs a; a.n = n; a.frame_count = frame_count;
    return staged(ctx, "predict_pts", {stage_in(a.state, state, SFIX * 8), stage_in(a.start_frame, start_frame, (size_t)n * 4), stage_in(a.num_obs, num_obs, (size_t)n * 4),
                                       stage_in(a.pt0, pt0, (size_t)n * 24), stage_in(a.depth, depth, (size_t)n * 8), stage_out(a.pts_cam, pts_cam, (size_t)n * 24),
                                       stage_out(a.valid, valid, (size_t)n)}, [&] {
        KERNEL(ctx, "predict_pts", (n + 127) / 128, 1, 128, 0, predict_pts_kernel, (a), for (int k = 0; k < n; k++) predict_pts_item(a, k));
    });
}

extern "C" int viwb_undistort_velocity(viwb_context *ctx, const viwb_pinhole *cam, int n, const float *pts, const float *prev_un_pts, const uint8_t *has_prev,
                                       double dt, float *un_pts, float *velocity) {
    if (!ctx || !cam || n < 0 || !pts || !un_pts) return VIWB_ERR_INVALID;
    const viwb_camera c = pinhole_camera(*cam);
    return viwb_undistort_velocity_camera(ctx, &c, n, pts, prev_un_pts, has_prev, dt, un_pts, velocity);
}

extern "C" int viwb_undistort_velocity_camera(viwb_context *ctx, const viwb_camera *cam, int n, const float *pts, const float *prev_un_pts, const uint8_t *has_prev,
                                              double dt, float *un_pts, float *velocity) {
    if (!ctx || n < 0 || !pts || !un_pts) return VIWB_ERR_INVALID;
    CamModel cm;
    if (camera_model(ctx, cam, &cm)) return VIWB_ERR_INVALID;
    if (n == 0) return VIWB_OK;
    UndistArgs a; a.n = n;
    a.fx = cm.fx; a.fy = cm.fy; a.cx = cm.cx; a.cy = cm.cy; a.k1 = cm.k1; a.k2 = cm.k2; a.p1 = cm.p1; a.p2 = cm.p2; a.dt = dt; a.model = cm.model; a.xi = cm.xi;
    return staged(ctx, "undistort", {stage_in(a.pts, pts, (size_t)n * 8), stage_in(a.prev_un, prev_un_pts, (size_t)n * 8), stage_in(a.has_prev, has_prev, (size_t)n),
                                     stage_out(a.un, un_pts, (size_t)n * 8), stage_out(a.vel, velocity, (size_t)n * 8)}, [&] {
        KERNEL(ctx, "undistort", (n + 127) / 128, 1, 128, 0, undistort_kernel, (a), for (int k = 0; k < n; k++) undistort_item(a, k));
    });
}

// -------------------------------------------------------------------------------------- feature tracker
extern "C" int viwb_lk_track(viwb_context *ctx, const uint8_t *prev_img, const uint8_t *next_img, int width, int height, int stride,
                             const float *prev_pts, float *next_pts, int n, int win_size, int max_level, int max_iter, float eps, int flags,
                             float min_eig_threshold, uint8_t *status, float *err) {
    if (!ctx || !prev_img || !next_img || !prev_pts || !next_pts || !status || n < 0 || width <= 0 || height <= 0) return VIWB_ERR_INVALID;
    if (win_size != 21) return fail(ctx, VIWB_ERR_UNSUPPORTED, "only the reference's 21x21 window is supported");
    if (max_level < 0 || max_level > 3) return fail(ctx, VIWB_ERR_UNSUPPORTED, "maxLevel must be 0..3");
    return lk_track_single(ctx, prev_img, next_img, width, height, stride, prev_pts, next_pts, n, max_level, max_iter, eps, flags, min_eig_threshold, status, err);
}

extern "C" int viwb_track_checked(viwb_context *ctx, const uint8_t *img_a, const uint8_t *img_b, int width, int height, int stride,
                                  const float *pts_a, float *pts_b, int n, int mode, int flow_back, uint8_t *status) {
    if (!ctx || !img_a || !img_b || !pts_a || !pts_b || !status || n < 0 || width <= 0 || height <= 0 || (mode != 0 && mode != 1)) return VIWB_ERR_INVALID;
    return lk_track_checked_single(ctx, img_a, img_b, width, height, stride, pts_a, pts_b, n, mode, flow_back, status);
}

extern "C" int viwb_lk_batch_create(viwb_context *ctx, int streams, int width, int height, int max_points, int stereo, int flow_back, viwb_lk_batch **out) {
    if (!ctx || !out || streams <= 0 || width <= 0 || height <= 0 || max_points <= 0) return VIWB_ERR_INVALID;
    return lk_batch_build(ctx, streams, width, height, max_points, stereo ? 1 : 0, flow_back ? 1 : 0, out);
}
extern "C" void viwb_lk_batch_destroy(viwb_lk_batch *b) { lk_batch_free(b); }
extern "C" int viwb_lk_batch_upload(viwb_lk_batch *b, const uint8_t *const *prev, const uint8_t *const *cur, const uint8_t *const *right, int stride,
                                    const float *prev_pts, const int32_t *n_prev, const float *stereo_pts, const int32_t *n_stereo) {
    if (!b || stride < b->w) return VIWB_ERR_INVALID;
    return lk_batch_upload(b, prev, cur, right, stride, prev_pts, n_prev, stereo_pts, n_stereo);
}
extern "C" int viwb_lk_batch_run(viwb_lk_batch *b) { return b ? lk_batch_execute(b, 3) : VIWB_ERR_INVALID; }
extern "C" int viwb_lk_batch_download(viwb_lk_batch *b, float *cur_pts, uint8_t *status, float *right_pts, uint8_t *status_right) {
    return b ? lk_batch_fetch(b, cur_pts, status, right_pts, status_right) : VIWB_ERR_INVALID;
}
extern "C" int viwb_set_mask(viwb_context *ctx, int width, int height, const float *pts, const int32_t *track_cnt, int n, int min_dist,
                             const uint8_t *base_mask, uint8_t *mask_out, int32_t *keep, int32_t *n_keep) {
    if (!ctx) return VIWB_ERR_INVALID;
    return det_set_mask(ctx, width, height, pts, track_cnt, n, min_dist, base_mask, mask_out, keep, n_keep);
}
extern "C" int viwb_good_features_to_track(viwb_context *ctx, const uint8_t *image, int width, int height, int stride, int max_corners, double quality_level,
                                           double min_distance, const uint8_t *mask, int mask_stride, float *corners, int capacity, int32_t *n_corners) {
    if (!ctx || stride < width || (mask && mask_stride < width)) return VIWB_ERR_INVALID;
    return det_good_features(ctx, image, width, height, stride, max_corners, quality_level, min_distance, mask, mask_stride, corners, capacity, n_corners);
}
extern "C" int viwb_detector_create(viwb_context *ctx, int streams, int width, int height, int max_pts, int min_dist, viwb_detector **out) {
    if (!ctx || !out) return VIWB_ERR_INVALID;
    return det_build(ctx, streams, width, height, max_pts, (double)min_dist, out);
}
extern "C" void viwb_detector_destroy(viwb_detector *d) { det_free(d); }
extern "C" int viwb_detector_detect(viwb_detector *d, const uint8_t *const *images, int stride, const viwb_lk_batch *resident, const uint8_t *const *base_masks,
                                    const float *pts, const int32_t *track_cnt, const int32_t *n_pts, int max_cnt, double quality_level,
                                    int32_t *keep, int32_t *n_keep, float *new_pts, int32_t *n_new, uint8_t *mask_out) {
    if (!d || !pts || !track_cnt || !n_pts || !keep || !n_keep || !new_pts || !n_new || (images && stride < d->w) || !(quality_level > 0.0)) return VIWB_ERR_INVALID;
    return det_detect(d, images, stride, resident, base_masks, pts, track_cnt, n_pts, max_cnt, quality_level, keep, n_keep, new_pts, n_new, mask_out);
}
extern "C" double viwb_detector_algorithmic_bytes(const viwb_detector *d) {
    if (!d) return 0.0;
    return (double)d->F * ((double)d->w * d->h + (double)d->maxn * (8 + 4 + 4 + 8));
}
extern "C" double viwb_lk_batch_algorithmic_bytes(const viwb_lk_batch *b) {
    if (!b) return 0.0;
    // per tick: read the new left (+right) level-0 images once, write their three coarser levels; points in/out
    double img = 0.0; for (int l = 0; l <= b->levels; l++) img += (double)b->lw[l] * b->lh[l];
    return (double)b->F * ((b->stereo ? 2.0 : 1.0) * img + (double)b->maxn * (b->stereo ? 2 : 1) * (8 + 8 + 1));
}
// page-lock caller-owned host buffers (camera frames) so that uploads run at full PCIe rate and asynchronously
extern "C" int viwb_tracker_create(viwb_context *ctx, int streams, int width, int height, const viwb_tracker_config *config, viwb_tracker **out) {
    if (!ctx || !out) return VIWB_ERR_INVALID;
    if (width < 3 || height < 3) return fail(ctx, VIWB_ERR_INVALID, "tracker: bad image size");
    viwb_camera cam[2] = {};
    if (config) for (int c = 0; c < 2; c++) cam[c] = pinhole_camera(config->cam[c]);
    return trk_build(ctx, streams, width, height, config, cam, out);
}
extern "C" int viwb_tracker_create_camera(viwb_context *ctx, int streams, int width, int height, const viwb_tracker_config *config, const viwb_camera cam[2],
                                          viwb_tracker **out) {
    if (!ctx || !out) return VIWB_ERR_INVALID;
    if (width < 3 || height < 3) return fail(ctx, VIWB_ERR_INVALID, "tracker: bad image size");
    return trk_build(ctx, streams, width, height, config, cam, out);
}
extern "C" void viwb_tracker_destroy(viwb_tracker *t) { trk_free(t); }
extern "C" int viwb_tracker_track(viwb_tracker *t, double cur_time, const uint8_t *const *left, const uint8_t *const *right, int stride, const float *predict_pts,
                                  const uint8_t *has_prediction) {
    if (!t) return VIWB_ERR_INVALID;
    if (stride < t->w) return fail(t->ctx, VIWB_ERR_INVALID, "tracker: stride smaller than the image width");
    if (predict_pts && !has_prediction) return fail(t->ctx, VIWB_ERR_INVALID, "tracker: predict_pts without has_prediction flags");
    return trk_track(t, cur_time, left, right, stride, predict_pts, has_prediction);
}
extern "C" int viwb_tracker_download(viwb_tracker *t, int32_t *n_left, int32_t *ids, int32_t *track_cnt, float *feat, int32_t *n_right, int32_t *ids_right,
                                     float *feat_right) {
    return t ? trk_fetch(t, n_left, ids, track_cnt, feat, n_right, ids_right, feat_right) : VIWB_ERR_INVALID;
}
extern "C" int viwb_tracker_feedback(viwb_tracker *t, const int32_t *n_remove, const int32_t *remove_ids, const int32_t *n_pred, const int32_t *pred_ids,
                                     const double *pred_pts_cam, const uint8_t *has_prediction) {
    return t ? trk_feedback_run(t, n_remove, remove_ids, n_pred, pred_ids, pred_pts_cam, has_prediction) : VIWB_ERR_INVALID;
}
extern "C" double viwb_tracker_algorithmic_bytes(const viwb_tracker *t) {
    if (!t) return 0.0;
    const viwb_lk_batch *b = t->lk;
    double px = 0; for (int l = 1; l <= b->levels; l++) px += (double)b->lw[l] * b->lh[l];
    const double img = (double)t->w * t->h, cams = t->stereo ? 2.0 : 1.0;
    return (double)t->F * (cams * (img + px) + img + (double)t->maxn * (cams * (24 + 4) + 4));
}
// -------------------------------------------------------------------------------------- resident FeatureManager (features_host.inl)
extern "C" int viwb_features_create(viwb_context *ctx, int streams, const viwb_features_config *config, viwb_features **out) {
    if (!ctx || !out) return VIWB_ERR_INVALID;
    return fm_build(ctx, streams, config, out);
}
extern "C" void viwb_features_destroy(viwb_features *fs) { fm_free(fs); }
extern "C" int viwb_features_add(viwb_features *fs, const int32_t *frame_count, const double *td, const int32_t *n_left, const int32_t *ids, const float *feat,
                                 const int32_t *n_right, const int32_t *ids_right, const float *feat_right) {
    return fs ? fm_add_host(fs, frame_count, td, n_left, ids, feat, n_right, ids_right, feat_right) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_add_tracked(viwb_features *fs, const viwb_tracker *t, const int32_t *frame_count, const double *td) {
    return fs ? fm_add_tracked(fs, t, frame_count, td) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_decisions(viwb_features *fs, int32_t *margin_flag, int32_t *last_track_num, int32_t *long_track_num, int32_t *new_feature_num,
                                       double *last_average_parallax) {
    return fs ? fm_decisions(fs, margin_flag, last_track_num, long_track_num, new_feature_num, last_average_parallax) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_triangulate(viwb_features *fs, const double *states) { return fs ? fm_triangulate_run(fs, states) : VIWB_ERR_INVALID; }
extern "C" int viwb_features_window(viwb_features *fs, int vis_cap, int32_t *num_landmarks, int32_t *num_vis, int32_t *vis_type, int32_t *vis_landmark,
                                    int32_t *vis_frame_i, int32_t *vis_frame_j, double *vis_obs, double *inv_depth, int32_t *landmark_ids) {
    return fs ? fm_window(fs, vis_cap, num_landmarks, num_vis, vis_type, vis_landmark, vis_frame_i, vis_frame_j, vis_obs, inv_depth, landmark_ids) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_set_depth(viwb_features *fs, const double *inv_depth) { return fs ? fm_set_depth_run(fs, inv_depth) : VIWB_ERR_INVALID; }
extern "C" int viwb_features_remove_outliers(viwb_features *fs, const uint8_t *outliers, int32_t *n_removed, int32_t *removed_ids) {
    return fs ? fm_remove_outliers(fs, outliers, n_removed, removed_ids) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_predict(viwb_features *fs, const double *states, const int32_t *frame_count, int32_t *n_pred, int32_t *pred_ids, double *pred_pts_cam,
                                     uint8_t *has_prediction) {
    return fs ? fm_predict_run(fs, states, frame_count, n_pred, pred_ids, pred_pts_cam, has_prediction) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_batch_create(viwb_features *fs, const viwb_problem *problems, const double *states, const viwb_options *options,
                                          const int32_t *margin_flags, int32_t *num_landmarks, viwb_batch **out) {
    return fs ? fm_batch_create(fs, problems, states, options, margin_flags, num_landmarks, out) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_set_depth_batch(viwb_features *fs, const viwb_batch *b) { return fs ? fm_set_depth_batch(fs, b) : VIWB_ERR_INVALID; }
extern "C" int viwb_features_remove_outliers_batch(viwb_features *fs, viwb_batch *b, double focal_length, double threshold_px, int32_t *n_removed,
                                                   int32_t *removed_ids) {
    return fs ? fm_remove_outliers_batch(fs, b, focal_length, threshold_px, n_removed, removed_ids) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_predict_batch(viwb_features *fs, const viwb_batch *b, const int32_t *frame_count, int32_t *n_pred, int32_t *pred_ids,
                                           double *pred_pts_cam, uint8_t *has_prediction) {
    return fs ? fm_predict_batch(fs, b, frame_count, n_pred, pred_ids, pred_pts_cam, has_prediction) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_slide(viwb_features *fs, const int32_t *frame_count, const uint8_t *shift_depth, const double *marg_R, const double *marg_P,
                                   const double *new_R, const double *new_P) {
    return fs ? fm_slide(fs, frame_count, shift_depth, marg_R, marg_P, new_R, new_P) : VIWB_ERR_INVALID;
}
extern "C" int viwb_features_remove_failures(viwb_features *fs) { return fs ? fm_remove_failures(fs) : VIWB_ERR_INVALID; }
extern "C" int viwb_features_download(viwb_features *fs, int32_t *n, int32_t *ids, int32_t *start_frame, int32_t *num_obs, double *depth, int32_t *solve_flag,
                                      float *obs, double *cur_td, uint8_t *is_stereo) {
    return fs ? fm_download(fs, n, ids, start_frame, num_obs, depth, solve_flag, obs, cur_td, is_stereo) : VIWB_ERR_INVALID;
}

extern "C" int viwb_host_register(viwb_context *ctx, void *ptr, size_t bytes) {
    bind_device(ctx);
    if (!ctx || !ptr) return VIWB_ERR_INVALID;
#ifndef VIWB_HOST_EMU
    CK((int)cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
#else
    (void)bytes;
#endif
    return VIWB_OK;
}
extern "C" int viwb_host_unregister(viwb_context *ctx, void *ptr) {
    bind_device(ctx);
    if (!ctx || !ptr) return VIWB_ERR_INVALID;
#ifndef VIWB_HOST_EMU
    CK((int)cudaHostUnregister(ptr));
#endif
    return VIWB_OK;
}
