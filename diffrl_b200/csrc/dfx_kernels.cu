// dfx_kernels.cu -- the C ABI (include/dfx.h) of the differentiable articulated rigid-body step and the
// LANE-GROUP sm_90a kernels (the humanoids and any generic articulation; the small DiffRL articulations run
// on the 32-environment tile kernels of dfx_tile.cu, same phase code, other mapping).
//
// Execution model here: a cooperative group of G lanes (8, 16 or 32; a sub-warp tile) owns one
// environment for the whole env-step; the environment's working set (transforms, spatial
// vectors, H^-1, adjoint accumulators: dfx_pack.h Layout) lives in a private shared-memory block,
// the model description is staged once per CTA into shared memory, and the only global traffic is
//   forward : q, qd, act [, musc] in   ->  q', qd' out  (+ the (q, qd) / H^-1 tape)
//   backward: cotangents of q', qd' + tape in  ->  cotangents of q, qd, act [, musc] out.
// Environments are env-major contiguous in global memory (the reference's State layout), so a
// group's loads are contiguous 60-120 B rows and a CTA's rows for one substep of the tape form
// one contiguous tile.  There is no dense contraction on this path: no tensor cores.
#include <cuda_runtime.h>

#include <atomic>
#include <cstring>
#include <string>

#include "dfx_launch.h"

namespace dfx {

template <int G_>
struct GroupCuda {
    static constexpr int G = G_;
    static constexpr bool kPathPasses = false;   // group barriers are cheap: level-by-level tree recursions
    static constexpr bool kFusedPhases = false;  // (merging phases saves CTA-wide barriers: nothing to gain with group-level ones)
    int lane;
    unsigned mask;
    __device__ __forceinline__ void sync() const { __syncwarp(mask); }
    bool psync;
    __device__ __forceinline__ void phase_sync() const { if (psync) __syncthreads(); }
    __device__ __forceinline__ void atomic_or(unsigned* p, unsigned v) const { atomicOr(p, v); }
    // one word of the fixed-point scatter-add (dfx_phases.h): native ATOMS.ADD, result unused -> fire and forget
    __device__ __forceinline__ void fx_add(int* p, int v) const { atomicAdd(p, v); }
    // fp32 add on shared memory: an ATOMS.CAST.SPIN loop, used only where contention is a few lanes at most
    __device__ __forceinline__ void atomic_add(float* p, float v) const { atomicAdd(p, v); }
    __device__ __forceinline__ float group_max(float v, float* slot) const {
        (void)slot;
#pragma unroll
        for (int o = G_ / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(mask, v, o, G_));
        return v;
    }
    // CTA-wide task loop (dfx_phases.h level_tasks): (k, env) pairs, k-major, over the threads of the CTA.  The
    // leading barrier publishes what the lane groups wrote with tile-level syncs only; the trailing one hands
    // the results back.  Co-resident CTAs start their task warps on different schedulers (rot).
    float* scratch0;
    int stride, envs_shift;
    bool cta_mode;
    template <class F>
    __device__ __forceinline__ void cta_tasks(float* s, int n, bool lead, F f) const {
        if (!cta_mode) {
            for (int k = lane; k < n; k += G_) f(s, k);
            __syncwarp(mask);
            return;
        }
        if (lead) __syncthreads();
        const int total = n << envs_shift;
        int t = (int)threadIdx.x - (int)(((blockIdx.x & 3u) << 5) & (blockDim.x - 1));   // blockDim.x is 32, 64 or 128
        if (t < 0) t += blockDim.x;
        for (; t < total; t += blockDim.x) {
            const int k = t >> envs_shift, e = t - (k << envs_shift);
            f(scratch0 + e * stride, k);
        }
        __syncthreads();
    }
    // cta_tasks() over the (k, env) pairs that satisfy pred(): the predicate is evaluated for all pairs (cheap),
    // the hits are compacted into a CTA-wide list (warp-aggregated atomic append), and f() then runs over the list
    // with full warps.  The order of the list varies from run to run; callers accumulate order-independently.
    int* task_count;     // [2] (double-buffered by phase parity is not needed: barriers separate uses)
    int* task_list;      // [n_max * envs]
    template <class Pr, class F>
    __device__ __forceinline__ void cta_compact(float* s, int n, Pr pred, F f) const {
        if (!cta_mode) {
            for (int k = lane; k < n; k += G_) if (pred(s, k)) f(s, k);
            __syncwarp(mask);
            return;
        }
        if (threadIdx.x == 0) *task_count = 0;
        __syncthreads();
        const int total = n << envs_shift;
        const int lane32 = threadIdx.x & 31;
        for (int t0 = (int)threadIdx.x - lane32; t0 < total; t0 += blockDim.x) {   // warp-uniform trip count
            const int t = t0 + lane32;
            bool hit = false;
            if (t < total) { const int k = t >> envs_shift, e = t - (k << envs_shift); hit = pred(scratch0 + e * stride, k); }
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (m) {
                int base = 0;
                if (lane32 == 0) base = atomicAdd(task_count, __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (hit) task_list[base + __popc(m & ((1u << lane32) - 1u))] = t;
            }
        }
        __syncthreads();
        const int hits = *task_count;
        int i = (int)threadIdx.x - (int)(((blockIdx.x & 3u) << 5) & (blockDim.x - 1));
        if (i < 0) i += blockDim.x;
        for (; i < hits; i += blockDim.x) {
            const int t = task_list[i];
            const int k = t >> envs_shift, e = t - (k << envs_shift);
            f(scratch0 + e * stride, k);
        }
        __syncthreads();
    }
    static constexpr bool kConcurrentItems = false;
    template <class Pr, class F, class H>
    __device__ __forceinline__ void cta_compact_with(float* s, int n, Pr pred, F f, int m, H item) const {
        for (int k = lane; k < m; k += G_) item(s, k);
        __syncwarp(mask);
        cta_compact(s, n, pred, f);
    }
    // tape blocks [b][env][n]: rows (n % 4 == 0, 16-byte aligned) move with cp.async (LDGSTS) / float4, one commit
    // group per row; the H^-1 blocks (n = D * D, any alignment) with plain loads
    __device__ __forceinline__ void block_in(float* dst, const float* base, long long b, int N, int env, int n, bool rows) const {
        const float* src = base + (b * N + env) * n;
        if (rows) {
            const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
            for (int i = lane * 4; i < n; i += G_ * 4)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + i * 4), "l"(src + i) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
        } else {
            for (int i = lane; i < n; i += G_) dst[i] = src[i];
        }
    }
    __device__ __forceinline__ void block_out(float* base, long long b, int N, int env, const float* src, int n, bool rows) const {
        float* dst = base + (b * N + env) * n;
        if (rows) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4* d4 = reinterpret_cast<float4*>(dst);
            for (int i = lane; i < n / 4; i += G_) d4[i] = s4[i];
        } else {
            for (int i = lane; i < n; i += G_) dst[i] = src[i];
        }
    }
    __device__ __forceinline__ void block_out_part(float* base, long long b, int N, int env, const float* src, const RowFmt& f, const float* stage, bool first, bool fenced = false) const {
        (void)stage; (void)fenced;
        if (!first) block_out(base, b, N, env, src, f.n, true);     // no asynchronous stores here: the whole row at once (always fp32)
    }
    __device__ __forceinline__ void row_unpack(float* dst, float* stage, const RowFmt& f) const { (void)dst; (void)stage; (void)f; }
    __device__ __forceinline__ void pre_store() const {}
    __device__ __forceinline__ void store_sync() const { __syncwarp(mask); }      // the group's row copy before integrate overwrites q, qd
    __device__ __forceinline__ void row_reusable() const {}
    __device__ __forceinline__ void finish() const {}
    static constexpr bool kBulkRows = false;
    __device__ __forceinline__ HinvView hinv_view(const float* base, long long b, int N, int env, int n) const { return HinvView{base + (b * N + env) * n, 1}; }
    // (rows are 60-120 B here and the head is not 16-byte aligned: one part, issued with the first call)
    __device__ __forceinline__ void row_in(float* dst, const float* base, long long b, int N, int env, int n, int head, int tail, bool first) const {
        (void)head; (void)tail;
        if (first) block_in(dst, base, b, N, env, n, true);
    }
    __device__ __forceinline__ void copy_wait_first() const { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
    __device__ __forceinline__ void copy_wait_all() const { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
};

// SL..SM > 0: model sizes known at compile time (the six DiffRL articulations are pre-instantiated); the scratch
// layout and every loop bound then fold into immediates.  SL == 0: generic run-time sizes.
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_step_kernel(const __grid_constant__ KernelArgs ka) {
    extern __shared__ __align__(16) float smem[];
    // ---- stage the model description
    float* fpack = smem;
    int* ipack = reinterpret_cast<int*>(smem + ((ka.blob.n_floats + 3) & ~3));
    for (int i = threadIdx.x; i < ka.blob.n_floats; i += blockDim.x) fpack[i] = ka.blob.floats[i];
    for (int i = threadIdx.x; i < ka.blob.n_ints; i += blockDim.x) ipack[i] = ka.blob.ints[i];
    __syncthreads();
    Pack P = bind_pack(ka.header, ka.blob, ipack, fpack);
    Layout Y = ka.layout;
    if constexpr (SL > 0) {
        P.L = SL; P.D = SD; P.Q = SQ; P.C = SC; P.M = SM;
        constexpr Layout kY = make_layout(SL, SD, SQ, SC, SM);
        Y = kY;
    }

    const int kEnvsPerCta = blockDim.x / G;
    const int local = threadIdx.x / G;
    // groups past the end redo the last environment (identical values are stored twice) so that every
    // thread of the CTA reaches the CTA-wide phase barriers
    int env = blockIdx.x * kEnvsPerCta + local;
    if (env >= ka.step.N) env = ka.step.N - 1;
    const int lane_in_warp = threadIdx.x & 31;
    GroupCuda<G> g;
    g.lane = threadIdx.x % G;
    g.psync = (ka.step.flags & 2) != 0;
    g.mask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << ((lane_in_warp / G) * G));
    float* s = smem + ka.pack_smem_floats + ka.cta_area_floats + (size_t)local * ka.scratch_stride;
    g.scratch0 = smem + ka.pack_smem_floats + ka.cta_area_floats;
    g.task_count = reinterpret_cast<int*>(smem + ka.pack_smem_floats);
    g.task_list = g.task_count + 4;
    g.stride = ka.scratch_stride;
    g.envs_shift = 31 - __clz(kEnvsPerCta > 0 ? kEnvsPerCta : 1);
    g.cta_mode = (ka.step.flags & 8) != 0;
    if (BACKWARD) env_step_backward(P, Y, s, g, env, ka.step);
    else env_step_forward(P, Y, s, g, env, ka.step);
}

}  // namespace dfx

// =====================================================================================
// C ABI
// =====================================================================================
using namespace dfx;

struct dfx_pack {
    int bf16;        // tape rows keep their middle (the forward intermediates) as bf16 -- tile kernels only
    int tile;        // 0: lane-group kernels; E = 8 / 16 / 32: stepped by the E-environment tile kernels (dfx_tile.cu); fixes the tape layout
    PackHost host;
    int device;
    int* d_ints;
    float* d_floats;
    Pack header;
    PackBlob blob;
};

static std::atomic<long long> g_launches{0};
long long dfx_count_launch(void) { return g_launches.fetch_add(1); }
static int g_group = 0;
static int g_flags = 9;   // include/dfx.h dfx_set_flags: 2 phase barriers, 4 generic kernels, 8 CTA-wide task loops, 32 no tile kernels
static int g_tape_bf16 = 0;   // dfx_set_tape_dtype
static int g_tile_envs = 0;   // dfx_set_tile_envs: 0 = the widest tile kernel that exists for the articulation

static int tile_mode(int E, const Pack& h) {
    if (h.jmask & ~tile_joint_mask(h.L, h.D, h.Q, h.C, h.M)) return -1;     // a joint type the tile kernels of these sizes are not compiled for
    switch (E) {
        case 8: return dfx_tile_mode_e8(h.L, h.D, h.Q, h.C, h.M);
        case 16: return dfx_tile_mode_e16(h.L, h.D, h.Q, h.C, h.M);
        case 32: return dfx_tile_mode_e32(h.L, h.D, h.Q, h.C, h.M);
    }
    return -1;
}

static void set_err(char* err, int n, const std::string& m) {
    if (err && n > 0) { strncpy(err, m.c_str(), n - 1); err[n - 1] = 0; }
}

extern "C" {

const char* dfx_version(void) { return "diffrl_b200 dfx 0.2 (sm_90a)"; }
int dfx_tile_joint_mask(int L, int D, int Q, int C, int M) { return tile_joint_mask(L, D, Q, C, M); }
int dfx_abi_sizeof(int which) {
    switch (which) {
        case 0: return (int)sizeof(DfxModelDesc);
        case 1: return (int)sizeof(DfxDerived);
        case 2: return (int)sizeof(DfxWalkerParams);
        case 3: return (int)sizeof(DfxPlanarParams);
        case 4: return (int)sizeof(DfxActionMap);
        case 5: return (int)sizeof(DfxEnvTransition);
        case 6: return (int)sizeof(DfxEnvTransitionAdj);
    }
    return -1;
}
long long dfx_launch_count(void) { return g_launches.load(); }
int dfx_set_flags(int flags) { g_flags = flags; return 0; }
int dfx_set_tape_dtype(int bf16) { g_tape_bf16 = bf16 ? 1 : 0; return 0; }
int dfx_set_tile_envs(int envs) {
    if (envs != 0 && envs != 8 && envs != 16 && envs != 32) return 1;
    g_tile_envs = envs;
    return 0;
}
int dfx_set_group_size(int lanes) {
    if (lanes != 0 && lanes != 8 && lanes != 16 && lanes != 32) return 1;
    g_group = lanes;
    return 0;
}

dfx_pack_t* dfx_pack_create(const DfxModelDesc* desc, int device, char* err, int err_len) {
    if (!desc) { set_err(err, err_len, "null DfxModelDesc"); return nullptr; }
    dfx_pack* p = new dfx_pack();
    std::string msg;
    if (!build_pack(*desc, p->host, msg)) { set_err(err, err_len, msg); delete p; return nullptr; }
    if (p->host.int_off.size() != 26 || p->host.float_off.size() != 17) { set_err(err, err_len, "internal: pack field count"); delete p; return nullptr; }
    p->device = device;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaMalloc(&p->d_ints, p->host.ints.size() * sizeof(int) + 16);
    if (e == cudaSuccess) e = cudaMalloc(&p->d_floats, p->host.floats.size() * sizeof(float) + 16);
    if (e == cudaSuccess) e = cudaMemcpy(p->d_ints, p->host.ints.data(), p->host.ints.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(p->d_floats, p->host.floats.data(), p->host.floats.size() * sizeof(float), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { set_err(err, err_len, std::string("CUDA: ") + cudaGetErrorString(e)); delete p; return nullptr; }
    p->header = p->host.header;
    p->blob.ints = p->d_ints; p->blob.floats = p->d_floats;
    p->blob.n_ints = (int)p->host.ints.size(); p->blob.n_floats = (int)p->host.floats.size();
    for (int i = 0; i < 26; ++i) p->blob.int_off[i] = (int)p->host.int_off[i];
    for (int i = 0; i < 17; ++i) p->blob.float_off[i] = (int)p->host.float_off[i];
    // flag bit 5 (32) keeps a supported articulation on the lane-group kernels (A/B runs); fixed per pack because
    // the two kernel families lay the tape out differently
    p->tile = 0;
    if (!(g_flags & 32)) {
        // auto: the widest tile kernel that is not an A/B-only instantiation (mode bit 4); dfx_set_tile_envs picks any
        static const int kWidths[3] = {32, 16, 8};
        for (int k = 0; k < 3 && !p->tile; ++k) {
            const int E = kWidths[k];
            const int mode = tile_mode(E, p->header);
            if (mode >= 0 && (g_tile_envs == 0 ? !(mode & 16) : g_tile_envs == E)) p->tile = E;
        }
    }
    if (p->tile) p->host.set_layout_mode(tile_mode(p->tile, p->header) & 3);
    p->bf16 = (p->tile && g_tape_bf16) ? 1 : 0;
    return p;
}

void dfx_pack_destroy(dfx_pack_t* p) {
    if (!p) return;
    cudaFree(p->d_ints);
    cudaFree(p->d_floats);
    delete p;
}

int dfx_pack_query(const dfx_pack_t* p, int what) {
    switch (what) {
        case DFX_QUERY_LINKS: return p->header.L;
        case DFX_QUERY_DOFS: return p->header.D;
        case DFX_QUERY_COORDS: return p->header.Q;
        case DFX_QUERY_CONTACTS: return p->header.C;
        case DFX_QUERY_MUSCLES: return p->header.M;
        case DFX_QUERY_FWD_SCRATCH_FLOATS: return p->host.layout.fwd_size;
        case DFX_QUERY_BWD_SCRATCH_FLOATS: return p->host.layout_bwd.bwd_size;
        case DFX_QUERY_TAPE_ROW_FLOATS: return p->host.layout.tape_row;
        case DFX_QUERY_TAPE_ROW_UNITS: return dfx_row_units(p->host.layout.tape_row, p->header.L, p->header.D, p->bf16 != 0);
        case DFX_QUERY_TREE_DEPTH: return p->header.nlev;
        case DFX_QUERY_TAPE_TILE: return p->tile;
        case DFX_QUERY_TAPE_BF16: return p->bf16;
        case DFX_QUERY_JOINT_MASK: return p->header.jmask;
    }
    return -1;
}

int dfx_pack_set_gravity(dfx_pack_t* p, float gx, float gy, float gz, int ground) {
    p->header.gx = gx; p->header.gy = gy; p->header.gz = gz;
    p->header.ground = (ground && p->header.C > 0) ? 1 : 0;
    return 0;
}

// environments as laid out in the tape: tile kernels pad to whole tiles
static int tape_envs(const dfx_pack* p, int n) { return p->tile ? ((n + p->tile - 1) / p->tile) * p->tile : n; }

long long dfx_tape_floats(const dfx_pack_t* p, int n, int substeps, int mm_freq) {
    return tape_geom(p->header.L, p->header.Q, p->header.D, tape_envs(p, n), substeps, mm_freq, p->bf16 != 0).total;
}

}  // extern "C"

// launch geometry of one step kernel (host arithmetic only, also exported through dfx_launch_plan)
struct LaunchPlan {
    int scratch_stride, pack_bytes, cta_area_bytes, envs_per_cta, ctas_per_sm;
    size_t smem;
};
// CTA-wide area: task counter (16 bytes) + one list slot per (contact point, environment)
static int cta_area(const dfx_pack* p, int envs_per_cta) {
    return 16 + ((p->header.C * envs_per_cta * 4 + 15) & ~15);
}
static LaunchPlan plan_launch(const dfx_pack* p, int G, bool bwd) {
    LaunchPlan lp{};
    const int per_env = bwd ? p->host.layout_bwd.bwd_size : p->host.layout.fwd_size;
    // multiple of 4 floats (16-byte cp.async rows) that is not a multiple of 32 (bank spreading between groups)
    lp.scratch_stride = (per_env + 3) & ~3;
    if (lp.scratch_stride % 32 == 0) lp.scratch_stride += 4;
    lp.pack_bytes = (((p->blob.n_floats + 3) & ~3) + ((p->blob.n_ints + 3) & ~3)) * 4;
    // environments per CTA: the candidate (128, 64 or 32 threads) that keeps the most environments resident
    // per SM under the shared-memory (227 KB) and register (64 K) budgets; ties go to the larger CTA
    const int regs_per_thread = bwd ? 128 : 96;
    int best = -1;
    for (int threads = kMaxThreads; threads >= 32 && threads >= G; threads /= 2) {
        const int e = threads / G;
        const size_t bytes = (size_t)lp.pack_bytes + cta_area(p, e) + (size_t)e * lp.scratch_stride * sizeof(float) + 1024;
        if (bytes > 227 * 1024) continue;
        int ctas = (int)((227 * 1024) / bytes);
        const int by_regs = 65536 / (regs_per_thread * threads);
        if (by_regs < ctas) ctas = by_regs;
        if (ctas > 32) ctas = 32;
        if (ctas * e > best) { best = ctas * e; lp.envs_per_cta = e; lp.ctas_per_sm = ctas; }
    }
    lp.cta_area_bytes = cta_area(p, lp.envs_per_cta);
    lp.smem = (size_t)lp.pack_bytes + lp.cta_area_bytes + (size_t)lp.envs_per_cta * lp.scratch_stride * sizeof(float);
    return lp;
}

template <int G, bool BWD, int SL, int SD, int SQ, int SC, int SM>
static cudaError_t launch_impl(const dfx_pack* p, const StepArgs& step, cudaStream_t stream) {
    KernelArgs ka;
    ka.header = p->header;
    ka.blob = p->blob;
    ka.layout = BWD ? p->host.layout_bwd : p->host.layout;
    ka.step = step;
    const LaunchPlan lp = plan_launch(p, G, BWD);
    ka.scratch_stride = lp.scratch_stride;
    ka.pack_smem_floats = lp.pack_bytes / 4;
    ka.cta_area_floats = lp.cta_area_bytes / 4;
    const int envs_per_cta = lp.envs_per_cta;
    if (envs_per_cta == 0) return cudaErrorInvalidConfiguration;
    const size_t smem = lp.smem;
    auto kern = dfx_step_kernel<G, BWD, SL, SD, SQ, SC, SM>;
    // (the opt-in to > 48 KB of dynamic shared memory is per device: set it on every launch, it is cheap)
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (step.N + envs_per_cta - 1) / envs_per_cta;
    kern<<<grid, envs_per_cta * G, smem, stream>>>(ka);
    g_launches.fetch_add(1);
    return cudaGetLastError();
}

// dispatch on the model sizes: specialised instantiations for the DiffRL articulations, generic otherwise
template <int G, bool BWD>
static cudaError_t launch(const dfx_pack* p, const StepArgs& step, cudaStream_t stream) {
    const Pack& h = p->header;
#define DFX_SPECIAL(l, d, q, c, m) \
    if (h.L == l && h.D == d && h.Q == q && h.C == c && h.M == m) return launch_impl<G, BWD, l, d, q, c, m>(p, step, stream);
    if (!(g_flags & 4)) {
        if constexpr (G == 16) {               // the group width pick_group() chooses for these models
            DFX_SPECIAL(9, 14, 15, 25, 0)      // Ant
            DFX_SPECIAL(3, 2, 2, 0, 0)         // CartPole
            DFX_SPECIAL(6, 6, 6, 8, 0)         // Hopper
            DFX_SPECIAL(9, 9, 9, 16, 0)        // HalfCheetah
        }
        if constexpr (G == 32) {
            DFX_SPECIAL(22, 27, 28, 35, 0)     // Humanoid
            DFX_SPECIAL(11, 24, 29, 88, 152)   // SNU humanoid (lower body, 152 muscles)
        }
    }
#undef DFX_SPECIAL
    return launch_impl<G, BWD, 0, 0, 0, 0, 0>(p, step, stream);
}

static cudaError_t launch_tile(const dfx_pack* p, const StepArgs& step, bool backward, cudaStream_t stream) {
    KernelArgs ka;
    ka.header = p->header;
    ka.blob = p->blob;
    ka.step = step;
    int e = (int)cudaErrorInvalidConfiguration;
    switch (p->tile) {
        case 8: e = dfx_tile_launch_e8(&ka, backward, stream); break;
        case 16: e = dfx_tile_launch_e16(&ka, backward, stream); break;
        case 32: e = dfx_tile_launch_e32(&ka, backward, stream); break;
    }
    g_launches.fetch_add(1);
    return (cudaError_t)e;
}

static int pick_group(const dfx_pack* p) {
    if (g_group) return g_group;
    const int widest = p->header.D > p->header.L ? p->header.D : p->header.L;
    return widest <= 16 ? 16 : 32;
}

extern "C" {

int dfx_launch_plan(const dfx_pack_t* p, int backward, int out[6]) {
    if (!p || !out) return (int)cudaErrorInvalidValue;
    if (p->tile) {      // one CTA = a tile of E environments
        KernelArgs ka;
        ka.header = p->header;
        ka.blob = p->blob;
        const size_t smem = p->tile == 8 ? dfx_tile_smem_e8(&ka, backward) : p->tile == 16 ? dfx_tile_smem_e16(&ka, backward) : dfx_tile_smem_e32(&ka, backward);
        const Layout& Y = backward ? p->host.layout_bwd : p->host.layout;
        out[0] = 32; out[1] = p->tile; out[2] = (int)((227 * 1024) / (smem + 1024)); out[3] = (int)smem;
        out[4] = ((backward ? Y.bwd_size : Y.fwd_size) + 3) & ~3;
        out[5] = (int)smem - out[4] * p->tile * 4;
        return 0;
    }
    const int G = pick_group(p);
    const LaunchPlan lp = plan_launch(p, G, backward != 0);
    out[0] = G; out[1] = lp.envs_per_cta; out[2] = lp.ctas_per_sm; out[3] = (int)lp.smem;
    out[4] = lp.scratch_stride; out[5] = lp.pack_bytes + lp.cta_area_bytes;
    return 0;
}

static int run_step(const dfx_pack_t* p, StepArgs& a, bool backward, void* stream) {
    a.hinv_base = tape_geom(p->header.L, p->header.Q, p->header.D, tape_envs(p, a.N), a.substeps, a.mm_freq, p->bf16 != 0).hinv_base;
    a.tape_bf16 = p->bf16;
    a.flags = g_flags;
    cudaStream_t st = (cudaStream_t)stream;
    if (p->tile) return (int)launch_tile(p, a, backward, st);
    if (backward) {
        switch (pick_group(p)) {
            case 8: return (int)launch<8, true>(p, a, st);
            case 16: return (int)launch<16, true>(p, a, st);
            default: return (int)launch<32, true>(p, a, st);
        }
    }
    switch (pick_group(p)) {
        case 8: return (int)launch<8, false>(p, a, st);
        case 16: return (int)launch<16, false>(p, a, st);
        default: return (int)launch<32, false>(p, a, st);
    }
}

static bool bind_map(const dfx_pack_t* p, const DfxActionMap* m, StepArgs& a) {
    const int width = m->is_muscle ? p->header.M : p->header.D;
    if (m->num_act <= 0 || m->offset < 0 || m->offset + m->num_act > width || !m->strength) return false;
    a.map_num_act = m->num_act; a.map_offset = m->offset; a.map_muscle = m->is_muscle ? 1 : 0;
    a.map_pre_scale = m->pre_scale; a.map_pre_bias = m->pre_bias; a.map_drive_scale = m->drive_scale;
    a.strength = m->strength;
    return true;
}

int dfx_step_forward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                     const float* q, const float* qd, const float* act, const float* musc,
                     float* q_out, float* qd_out, float* tape, const DfxDerived* derived, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0) return (int)cudaErrorInvalidValue;
    if (!q || !qd || !act || !q_out || !qd_out || (p->header.M > 0 && !musc)) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.q = q; a.qd = qd; a.act = act; a.musc = musc; a.q_out = q_out; a.qd_out = qd_out; a.tape = tape;
    if (derived) { a.derived = *derived; a.has_derived = 1; }
    return run_step(p, a, false, stream);
}

int dfx_step_backward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                      const float* act, const float* musc, const float* tape,
                      const float* gq_out, const float* gqd_out,
                      float* gq, float* gqd, float* gact, float* gmusc, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !tape || !act) return (int)cudaErrorInvalidValue;
    if (p->header.M > 0 && !musc) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.act = act; a.musc = musc; a.tape_in = tape; a.gq_out = gq_out; a.gqd_out = gqd_out;
    a.gq = gq; a.gqd = gqd; a.gact = gact; a.gmusc = gmusc;
    return run_step(p, a, true, stream);
}

int dfx_step_forward_mapped(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                            const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                            float* used, float* q_out, float* qd_out, float* tape, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !q || !qd || !map || !raw || !q_out || !qd_out) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    if (!bind_map(p, map, a)) return (int)cudaErrorInvalidValue;
    if (!a.map_muscle && p->header.M > 0 && !act_other) return (int)cudaErrorInvalidValue;
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.q = q; a.qd = qd; a.raw = raw; a.used = used; a.q_out = q_out; a.qd_out = qd_out; a.tape = tape;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    return run_step(p, a, false, stream);
}

int dfx_step_backward_mapped(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                             const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                             const float* gq_out, const float* gqd_out, const float* g_used,
                             float* gq, float* gqd, float* g_raw, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !tape || !map || !raw) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    if (!bind_map(p, map, a)) return (int)cudaErrorInvalidValue;
    if (!a.map_muscle && p->header.M > 0 && !act_other) return (int)cudaErrorInvalidValue;
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.raw = raw; a.tape_in = tape; a.gq_out = gq_out; a.gqd_out = gqd_out; a.g_used = g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    return run_step(p, a, true, stream);
}

// ---- env.step() as one launch (include/dfx.h): the mapped step with the transition as epilogue (tile kernels), or the two
// launches back to back (lane-group kernels)
// the tile kernels stage the transition in dead scratch (dfx_env_dev.h tile_transition_*): is there enough of it?
static bool transition_fits(const dfx_pack_t* p, int kind, const DfxWalkerParams& w, const DfxPlanarParams& pl, bool backward) {
    if (!p->tile) return false;
    const int no = kind == 1 ? w.num_obs : pl.num_obs, na = kind == 1 ? w.num_act : pl.num_act;
    if (backward) return 2 * no + 3 * (p->header.Q + p->header.D + na) <= p->host.layout_bwd.bwd_size;
    return 2 * no + 1 <= p->host.layout.fwd_size - p->host.layout.act;
}

static bool transition_ok(int kind, const DfxWalkerParams& w, const DfxPlanarParams& pl, const dfx_pack_t* p, const DfxActionMap* m) {
    if (kind == 1) return w.num_q == p->header.Q && w.num_qd == p->header.D && w.num_act == m->num_act && w.num_obs > 0 && w.num_obs <= 96;
    if (kind == 2) return pl.num_q == p->header.Q && pl.num_qd == p->header.D && pl.num_act == m->num_act && pl.num_obs > 0 && pl.kind >= 0 && pl.kind <= 2;
    return false;
}

int dfx_env_step_forward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                         const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                         float* used, float* q_sim, float* qd_sim, float* tape, const DfxEnvTransition* tr, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !q || !qd || !map || !raw || !used || !q_sim || !qd_sim || !tr) return (int)cudaErrorInvalidValue;
    if (!transition_ok(tr->kind, tr->walker, tr->planar, p, map)) return (int)cudaErrorInvalidValue;
    if (!tr->progress || !tr->start_q || !tr->start_qd || !tr->obs_before || !tr->rew || !tr->reset || !tr->q_next || !tr->qd_next ||
        !tr->actions_next || !tr->progress_next || !tr->obs_next) return (int)cudaErrorInvalidValue;
    if (!transition_fits(p, tr->kind, tr->walker, tr->planar, false)) {
        const int e = dfx_step_forward_mapped(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, used, q_sim, qd_sim, tape, stream);
        if (e != 0) return e;
        return tr->kind == 1
            ? dfx_walker_transition_forward(&tr->walker, n, q_sim, qd_sim, used, tr->progress, tr->start_q, tr->start_qd, tr->obs_before, tr->rew,
                                            tr->reset, tr->q_next, tr->qd_next, tr->actions_next, tr->progress_next, tr->obs_next, stream)
            : dfx_planar_transition_forward(&tr->planar, n, q_sim, qd_sim, used, tr->progress, tr->start_q, tr->start_qd, tr->obs_before, tr->rew,
                                            tr->reset, tr->q_next, tr->qd_next, tr->actions_next, tr->progress_next, tr->obs_next, stream);
    }
    StepArgs a;
    memset(&a, 0, sizeof a);
    if (!bind_map(p, map, a)) return (int)cudaErrorInvalidValue;
    if (!a.map_muscle && p->header.M > 0 && !act_other) return (int)cudaErrorInvalidValue;
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.q = q; a.qd = qd; a.raw = raw; a.used = used; a.q_out = q_sim; a.qd_out = qd_sim; a.tape = tape;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    a.env_kind = tr->kind;
    a.env = *tr;
    return run_step(p, a, false, stream);
}

int dfx_env_step_backward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                          const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                          const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !tape || !map || !raw || !tr) return (int)cudaErrorInvalidValue;
    if (!transition_ok(tr->kind, tr->walker, tr->planar, p, map)) return (int)cudaErrorInvalidValue;
    if (!tr->q_sim || !tr->qd_sim || !tr->used || !tr->reset || !tr->gq_sim || !tr->gqd_sim || !tr->g_used) return (int)cudaErrorInvalidValue;
    if (!transition_fits(p, tr->kind, tr->walker, tr->planar, true)) {
        const int e = tr->kind == 1
            ? dfx_walker_transition_backward(&tr->walker, n, tr->q_sim, tr->qd_sim, tr->used, tr->reset, tr->g_obs_before, tr->g_rew, tr->g_q_next,
                                             tr->g_qd_next, tr->g_actions_next, tr->g_obs_next, tr->gq_sim, tr->gqd_sim, tr->g_used, stream)
            : dfx_planar_transition_backward(&tr->planar, n, tr->q_sim, tr->qd_sim, tr->used, tr->reset, tr->g_obs_before, tr->g_rew, tr->g_q_next,
                                             tr->g_qd_next, tr->g_actions_next, tr->g_obs_next, tr->gq_sim, tr->gqd_sim, tr->g_used, stream);
        if (e != 0) return e;
        return dfx_step_backward_mapped(p, n, substeps, mm_freq, dt, map, raw, act_other, tape, tr->gq_sim, tr->gqd_sim, tr->g_used, gq, gqd, g_raw, stream);
    }
    StepArgs a;
    memset(&a, 0, sizeof a);
    if (!bind_map(p, map, a)) return (int)cudaErrorInvalidValue;
    if (!a.map_muscle && p->header.M > 0 && !act_other) return (int)cudaErrorInvalidValue;
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    a.raw = raw; a.tape_in = tape; a.gq_out = tr->gq_sim; a.gqd_out = tr->gqd_sim; a.g_used = tr->g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    a.env_kind = tr->kind;
    a.env_adj = *tr;
    return run_step(p, a, true, stream);
}

// ---- recompute adjoint (include/dfx.h dfx_*_backward_recompute): no stored tape, the env-step's forward is re-run from its
// input state into a one-env-step workspace right before the adjoint reads it
long long dfx_recompute_workspace_floats(const dfx_pack_t* p, int n, int substeps, int mm_freq) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0) return -1;
    return dfx_tape_floats(p, n, substeps, mm_freq) + (long long)n * (p->header.Q + p->header.D);
}

// end state of the recomputed forward: the workspace's tail, q [n*Q] then qd [n*D]
static float* workspace_q_end(const dfx_pack_t* p, const StepArgs& a, float* ws) { return ws + dfx_tape_floats(p, a.N, a.substeps, a.mm_freq); }

// one launch on the tile kernels: the forward into the workspace, the barrier sequence of dfx_tile_recompute_kernel, the adjoint.
// `a` holds the adjoint's arguments (as the stored-tape entry would launch them); the forward's are added here.
static int run_recompute_fused(const dfx_pack_t* p, StepArgs& a, const float* q, const float* qd, float* ws, void* stream) {
    a.q = q; a.qd = qd;
    a.q_out = workspace_q_end(p, a, ws); a.qd_out = a.q_out + (long long)a.N * p->header.Q;
    a.tape = ws; a.tape_in = ws;
    a.used = nullptr; a.has_derived = 0;
    a.hinv_base = tape_geom(p->header.L, p->header.Q, p->header.D, tape_envs(p, a.N), a.substeps, a.mm_freq, p->bf16 != 0).hinv_base;
    a.tape_bf16 = p->bf16;
    a.flags = g_flags;
    KernelArgs ka;
    ka.header = p->header;
    ka.blob = p->blob;
    ka.step = a;
    int e = (int)cudaErrorInvalidConfiguration;
    switch (p->tile) {
        case 8: e = dfx_tile_launch_recompute_e8(&ka, stream); break;
        case 16: e = dfx_tile_launch_recompute_e16(&ka, stream); break;
        case 32: e = dfx_tile_launch_recompute_e32(&ka, stream); break;
    }
    g_launches.fetch_add(1);
    return e;
}

// the fused kernel exists for every tile pack; the A/B variants of flag bit 6 have none (two launches instead)
static bool recompute_fuses(const dfx_pack_t* p) { return p->tile != 0 && !(g_flags & 64); }

int dfx_step_backward_recompute(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                const float* q, const float* qd, const float* act, const float* musc, float* workspace,
                                const float* gq_out, const float* gqd_out,
                                float* gq, float* gqd, float* gact, float* gmusc, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !q || !qd || !workspace || !act) return (int)cudaErrorInvalidValue;
    if (p->header.M > 0 && !musc) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    if (!recompute_fuses(p)) {
        float* q_end = workspace_q_end(p, a, workspace);
        const int e = dfx_step_forward(p, n, substeps, mm_freq, dt, q, qd, act, musc, q_end, q_end + (long long)n * p->header.Q, workspace, nullptr, stream);
        if (e != 0) return e;
        return dfx_step_backward(p, n, substeps, mm_freq, dt, act, musc, workspace, gq_out, gqd_out, gq, gqd, gact, gmusc, stream);
    }
    a.act = act; a.musc = musc; a.gq_out = gq_out; a.gqd_out = gqd_out;
    a.gq = gq; a.gqd = gqd; a.gact = gact; a.gmusc = gmusc;
    return run_recompute_fused(p, a, q, qd, workspace, stream);
}

int dfx_step_backward_mapped_recompute(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                       const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                       float* workspace, const float* gq_out, const float* gqd_out, const float* g_used,
                                       float* gq, float* gqd, float* g_raw, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !q || !qd || !workspace || !map || !raw) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    if (!bind_map(p, map, a)) return (int)cudaErrorInvalidValue;
    if (!a.map_muscle && p->header.M > 0 && !act_other) return (int)cudaErrorInvalidValue;
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    if (!recompute_fuses(p)) {
        float* q_end = workspace_q_end(p, a, workspace);
        const int e = dfx_step_forward_mapped(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, nullptr, q_end,
                                              q_end + (long long)n * p->header.Q, workspace, stream);
        if (e != 0) return e;
        return dfx_step_backward_mapped(p, n, substeps, mm_freq, dt, map, raw, act_other, workspace, gq_out, gqd_out, g_used, gq, gqd, g_raw, stream);
    }
    a.raw = raw; a.gq_out = gq_out; a.gqd_out = gqd_out; a.g_used = g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    return run_recompute_fused(p, a, q, qd, workspace, stream);
}

int dfx_env_step_backward_recompute(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                    const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                    float* workspace, const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || !q || !qd || !workspace || !map || !raw || !tr) return (int)cudaErrorInvalidValue;
    if (!transition_ok(tr->kind, tr->walker, tr->planar, p, map)) return (int)cudaErrorInvalidValue;
    if (!tr->q_sim || !tr->qd_sim || !tr->used || !tr->reset || !tr->gq_sim || !tr->gqd_sim || !tr->g_used) return (int)cudaErrorInvalidValue;
    StepArgs a;
    memset(&a, 0, sizeof a);
    if (!bind_map(p, map, a)) return (int)cudaErrorInvalidValue;
    if (!a.map_muscle && p->header.M > 0 && !act_other) return (int)cudaErrorInvalidValue;
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    if (!recompute_fuses(p) || !transition_fits(p, tr->kind, tr->walker, tr->planar, true)) {
        // the plain mapped forward (the transition's outputs are not needed again: its adjoint reads tr->q_sim, ...), then the
        // stored-tape entry, which runs the transition adjoint as its prologue or as a launch of its own
        float* q_end = workspace_q_end(p, a, workspace);
        const int e = dfx_step_forward_mapped(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, nullptr, q_end,
                                              q_end + (long long)n * p->header.Q, workspace, stream);
        if (e != 0) return e;
        return dfx_env_step_backward(p, n, substeps, mm_freq, dt, map, raw, act_other, workspace, tr, gq, gqd, g_raw, stream);
    }
    a.raw = raw; a.gq_out = tr->gq_sim; a.gqd_out = tr->gqd_sim; a.g_used = tr->g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    a.env_kind = tr->kind;
    a.env_adj = *tr;
    return run_recompute_fused(p, a, q, qd, workspace, stream);
}

}  // extern "C"
