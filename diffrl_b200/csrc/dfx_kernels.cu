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
// (instantiated twice: without and with the external wrench (WRENCH; include/dfx.h DfxExternalWrench) -- two kernels of their
//  own, so that the ones without keep their code)
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM, bool WRENCH>
__device__ __forceinline__ void step_kernel_body(const KernelArgs& ka) {
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
    if (BACKWARD) env_step_backward<WRENCH>(P, Y, s, g, env, ka.step, ka.wrench);
    else env_step_forward<WRENCH>(P, Y, s, g, env, ka.step, ka.wrench);
}

template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_step_kernel(const __grid_constant__ KernelArgs ka) {
    step_kernel_body<G, BACKWARD, SL, SD, SQ, SC, SM, false>(ka);
}
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_step_wrench_kernel(const __grid_constant__ KernelArgs ka) {
    step_kernel_body<G, BACKWARD, SL, SD, SQ, SC, SM, true>(ka);
}

// Link state (include/dfx.h dfx_link_state_forward / _backward; dfx_step.h link_state_*): the set-up of step_kernel_body, then the
// kinematics of (q, qd) or their adjoint in the step's forward / backward layout.  The pointers come as a kernel parameter of their
// own (KernelArgs stays as the step kernels have it).
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_link_state_kernel(const __grid_constant__ KernelArgs ka,
                                                                    const __grid_constant__ LinkStateArgs la) {
    extern __shared__ __align__(16) float smem[];
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
    int env = blockIdx.x * kEnvsPerCta + local;      // (groups past the end redo the last environment, as in step_kernel_body)
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
    if (BACKWARD) link_state_backward(P, Y, s, g, env, la);
    else link_state_forward(P, Y, s, g, env, la);
}

// Contact state (include/dfx.h dfx_contact_state_forward / _backward; dfx_step.h contact_state_*): the set-up of
// dfx_link_state_kernel line for line (keep the two in step), then the ground-contact model at (q, qd) or its adjoint.  (One kernel
// templated on the readout would rename the link-state kernels and change their code: the set-up is written out per kernel.)
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_contact_state_kernel(const __grid_constant__ KernelArgs ka,
                                                                      const __grid_constant__ ContactStateArgs ca) {
    extern __shared__ __align__(16) float smem[];
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
    int env = blockIdx.x * kEnvsPerCta + local;      // (groups past the end redo the last environment, as in step_kernel_body)
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
    if (BACKWARD) contact_state_backward(P, Y, s, g, env, ca);
    else contact_state_forward(P, Y, s, g, env, ca);
}

// Dynamics state (include/dfx.h dfx_dynamics_state_forward / _backward; dfx_step.h dynamics_state_*): the set-up of
// dfx_link_state_kernel line for line (keep the two in step), then the first substep's dynamics, or their seeded adjoint on the
// one-substep tape that dfx_step_forward_ex wrote into the workspace (ka.step.tape_in) in the launch before.
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_dynamics_state_kernel(const __grid_constant__ KernelArgs ka,
                                                                       const __grid_constant__ DynamicsStateArgs da) {
    extern __shared__ __align__(16) float smem[];
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
    int env = blockIdx.x * kEnvsPerCta + local;      // (groups past the end redo the last environment, as in step_kernel_body)
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
    if (BACKWARD) dynamics_state_backward(P, Y, s, g, env, ka.step, da);
    else dynamics_state_forward(P, Y, s, g, env, da);
}

// Jacobian state (include/dfx.h dfx_jacobian_state_forward / _backward; dfx_step.h jacobian_state_*): the set-up of
// dfx_link_state_kernel line for line (keep the two in step), then the kinematics of (q, qd) and the stores of J and body_a_s, or
// their adjoint.
template <int G, bool BACKWARD, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(kMaxThreads) dfx_jacobian_state_kernel(const __grid_constant__ KernelArgs ka,
                                                                       const __grid_constant__ JacobianStateArgs ja) {
    extern __shared__ __align__(16) float smem[];
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
    int env = blockIdx.x * kEnvsPerCta + local;      // (groups past the end redo the last environment, as in step_kernel_body)
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
    if (BACKWARD) jacobian_state_backward(P, Y, s, g, env, ja);
    else jacobian_state_forward(P, Y, s, g, env, ja);
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
    int* d_corder;   // [C]: Model index of the pack's contact n (the contact state's outputs are in the Model's order)
    Pack header;
    PackBlob blob;
};

static std::atomic<long long> g_launches{0};
long long dfx_count_launch(void) { return g_launches.fetch_add(1); }
static int g_group = 0;
static int g_flags = 9;   // include/dfx.h dfx_set_flags: 2 phase barriers, 4 generic kernels, 8 CTA-wide task loops, 32 no tile kernels
static int g_tape_bf16 = 0;   // dfx_set_tape_dtype
static int g_tile_envs = 0;   // dfx_set_tile_envs: 0 = the widest tile kernel that exists for the articulation

// the tile kernels of width E = 8, 16 or 32 (dfx_tile.cu)
static const DfxTileApi* tile_api(int E) {
    switch (E) {
        case 8: return dfx_tile_api_e8();
        case 16: return dfx_tile_api_e16();
        case 32: return dfx_tile_api_e32();
    }
    return nullptr;
}

static int tile_mode(int E, const Pack& h) {
    if (h.jmask & ~tile_joint_mask(h.L, h.D, h.Q, h.C, h.M)) return -1;     // a joint type the tile kernels of these sizes are not compiled for
    return tile_api(E)->mode(h.L, h.D, h.Q, h.C, h.M);
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
        case 7: return (int)sizeof(DfxExternalWrench);
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
    if (e == cudaSuccess) e = cudaMalloc(&p->d_corder, p->host.corder.size() * sizeof(int) + 16);
    if (e == cudaSuccess && !p->host.corder.empty())
        e = cudaMemcpy(p->d_corder, p->host.corder.data(), p->host.corder.size() * sizeof(int), cudaMemcpyHostToDevice);
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
    cudaFree(p->d_corder);
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
// wrench: the external-wrench kernels, whose scratch ends past the layout's (dfx_pack.h wrench_scratch_end)
static LaunchPlan plan_launch(const dfx_pack* p, int G, bool bwd, bool wrench = false) {
    LaunchPlan lp{};
    // multiple of 4 floats (16-byte cp.async rows) that is not a multiple of 32 (bank spreading between groups)
    lp.scratch_stride = scratch_floats(bwd ? p->host.layout_bwd : p->host.layout, p->header.L, bwd, wrench);
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

// the kernel argument block of a launch; the launch functions add the layout and the scratch geometry
static KernelArgs kernel_args(const dfx_pack* p, const StepArgs& step, const DfxExternalWrench* w) {
    KernelArgs ka;
    ka.header = p->header;
    ka.blob = p->blob;
    ka.step = step;
    ka.wrench = w ? *w : DfxExternalWrench{nullptr, nullptr};
    return ka;
}

// a tile launch is counted whatever the tile function returns (also when it refuses, e.g. a wrench under flag bit 6)
static int counted(int e) {
    g_launches.fetch_add(1);
    return e;
}

// the lane-group kernel families
enum GroupFamily { kStep, kStepWrench, kLinkState, kContactState, kDynamicsState, kJacobianState };

// one lane-group launch: the family's kernel of group width G, size-specialised (SL..SM > 0) or generic, with plan_launch's
// geometry; ra: the readout's kernel parameter (a LinkStateArgs, ContactStateArgs, DynamicsStateArgs or JacobianStateArgs), NULL
// for the step families.  The external-wrench step and the dynamics state keep the wrench past the layout's end.
template <GroupFamily F, int G, bool BWD, int SL, int SD, int SQ, int SC, int SM>
static cudaError_t launch_impl(const dfx_pack* p, KernelArgs& ka, const void* ra, cudaStream_t stream) {
    ka.layout = BWD ? p->host.layout_bwd : p->host.layout;
    const LaunchPlan lp = plan_launch(p, G, BWD, F == kStepWrench || F == kDynamicsState);
    ka.scratch_stride = lp.scratch_stride;
    ka.pack_smem_floats = lp.pack_bytes / 4;
    ka.cta_area_floats = lp.cta_area_bytes / 4;
    if (lp.envs_per_cta == 0) return cudaErrorInvalidConfiguration;
    const int grid = (ka.step.N + lp.envs_per_cta - 1) / lp.envs_per_cta;
    const auto go = [&](auto kern, const auto&... extra) {
        // (the opt-in to > 48 KB of dynamic shared memory is per device: set it on every launch, it is cheap)
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lp.smem);
        if (e != cudaSuccess) return e;
        kern<<<grid, lp.envs_per_cta * G, lp.smem, stream>>>(ka, extra...);
        g_launches.fetch_add(1);
        return cudaGetLastError();
    };
    if constexpr (F == kLinkState) {
        return go(dfx_link_state_kernel<G, BWD, SL, SD, SQ, SC, SM>, *static_cast<const LinkStateArgs*>(ra));
    } else if constexpr (F == kContactState) {
        return go(dfx_contact_state_kernel<G, BWD, SL, SD, SQ, SC, SM>, *static_cast<const ContactStateArgs*>(ra));
    } else if constexpr (F == kDynamicsState) {
        return go(dfx_dynamics_state_kernel<G, BWD, SL, SD, SQ, SC, SM>, *static_cast<const DynamicsStateArgs*>(ra));
    } else if constexpr (F == kJacobianState) {
        return go(dfx_jacobian_state_kernel<G, BWD, SL, SD, SQ, SC, SM>, *static_cast<const JacobianStateArgs*>(ra));
    } else {
        // (the step kernel is referenced before its external-wrench twin, in every instantiation: nvcc emits the kernels in the
        //  order they are first referenced, and the code of some depends on that order)
        auto kern = dfx_step_kernel<G, BWD, SL, SD, SQ, SC, SM>;
        if constexpr (F == kStepWrench) kern = dfx_step_wrench_kernel<G, BWD, SL, SD, SQ, SC, SM>;
        return go(kern);
    }
}

// the size-specialised lane-group instantiations (the six DiffRL articulations), by the group width pick_group() chooses for them
#define DFX_GROUP_SPECIALS_16(X)                                                                     \
    X(9, 14, 15, 25, 0)      /* Ant */                                                               \
    X(3, 2, 2, 0, 0)         /* CartPole */                                                          \
    X(6, 6, 6, 8, 0)         /* Hopper */                                                            \
    X(9, 9, 9, 16, 0)        /* HalfCheetah */
#define DFX_GROUP_SPECIALS_32(X)                                                                     \
    X(22, 27, 28, 35, 0)     /* Humanoid */                                                          \
    X(11, 24, 29, 88, 152)   /* SNU humanoid (lower body, 152 muscles) */

// dispatch on the model sizes: specialised instantiations for the DiffRL articulations, generic otherwise (and under flag bit 2)
template <GroupFamily F, int G, bool BWD>
static cudaError_t launch(const dfx_pack* p, KernelArgs& ka, const void* ra, cudaStream_t stream) {
    const Pack& h = p->header;
#define DFX_SPECIAL(l, d, q, c, m) \
    if (h.L == l && h.D == d && h.Q == q && h.C == c && h.M == m) return launch_impl<F, G, BWD, l, d, q, c, m>(p, ka, ra, stream);
    if (!(g_flags & 4)) {
        if constexpr (G == 16) { DFX_GROUP_SPECIALS_16(DFX_SPECIAL) }
        if constexpr (G == 32) { DFX_GROUP_SPECIALS_32(DFX_SPECIAL) }
    }
#undef DFX_SPECIAL
    return launch_impl<F, G, BWD, 0, 0, 0, 0, 0>(p, ka, ra, stream);
}

static int pick_group(const dfx_pack* p) {
    if (g_group) return g_group;
    const int widest = p->header.D > p->header.L ? p->header.D : p->header.L;
    return widest <= 16 ? 16 : 32;
}

// the lane-group kernels of pick_group()'s width
template <GroupFamily F>
static int run_group(const dfx_pack_t* p, KernelArgs& ka, bool backward, const void* ra, cudaStream_t st) {
    switch (pick_group(p)) {
        case 8: return (int)(backward ? launch<F, 8, true>(p, ka, ra, st) : launch<F, 8, false>(p, ka, ra, st));
        case 16: return (int)(backward ? launch<F, 16, true>(p, ka, ra, st) : launch<F, 16, false>(p, ka, ra, st));
        default: return (int)(backward ? launch<F, 32, true>(p, ka, ra, st) : launch<F, 32, false>(p, ka, ra, st));
    }
}

// ---- the step entries: one set of argument checks and one StepArgs builder behind all of them

// the checks every step entry starts with, and StepArgs with the env-step's sizes (false: cudaErrorInvalidValue)
static bool step_args(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt, const DfxExternalWrench* w, StepArgs& a) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0 || (w && !w->f_ext)) return false;
    memset(&a, 0, sizeof a);
    a.N = n; a.substeps = substeps; a.mm_freq = mm_freq;
    a.dt_sub = (float)(dt / (double)substeps);
    return true;
}

// the action map of the mapped entries, and act_other: the actuation the map does not form (muscle activations under a joint map,
// which an articulation with muscles needs; joint actuation under a muscle map, or none)
static bool bind_map(const dfx_pack_t* p, const DfxActionMap* m, const float* act_other, StepArgs& a) {
    const int width = m->is_muscle ? p->header.M : p->header.D;
    if (m->num_act <= 0 || m->offset < 0 || m->offset + m->num_act > width || !m->strength) return false;
    if (!m->is_muscle && p->header.M > 0 && !act_other) return false;
    a.map_num_act = m->num_act; a.map_offset = m->offset; a.map_muscle = m->is_muscle ? 1 : 0;
    a.map_pre_scale = m->pre_scale; a.map_pre_bias = m->pre_bias; a.map_drive_scale = m->drive_scale;
    a.strength = m->strength;
    if (a.map_muscle) a.act = act_other; else a.musc = act_other;
    return true;
}

// the transition of the env-step entries: its sizes match the pack and the action map, and its rows are given
static bool transition_sizes_ok(int kind, const DfxWalkerParams& w, const DfxPlanarParams& pl, const dfx_pack_t* p, const DfxActionMap* m) {
    if (kind == 1) return w.num_q == p->header.Q && w.num_qd == p->header.D && w.num_act == m->num_act && w.num_obs > 0 && w.num_obs <= 96;
    if (kind == 2) return pl.num_q == p->header.Q && pl.num_qd == p->header.D && pl.num_act == m->num_act && pl.num_obs > 0 && pl.kind >= 0 && pl.kind <= 2;
    return false;
}
static bool transition_ok(const dfx_pack_t* p, const DfxActionMap* m, const DfxEnvTransition* tr) {
    return tr && transition_sizes_ok(tr->kind, tr->walker, tr->planar, p, m) && tr->progress && tr->start_q && tr->start_qd && tr->obs_before &&
           tr->rew && tr->reset && tr->q_next && tr->qd_next && tr->actions_next && tr->progress_next && tr->obs_next;
}
static bool transition_ok(const dfx_pack_t* p, const DfxActionMap* m, const DfxEnvTransitionAdj* tr) {
    return tr && transition_sizes_ok(tr->kind, tr->walker, tr->planar, p, m) && tr->q_sim && tr->qd_sim && tr->used && tr->reset && tr->gq_sim &&
           tr->gqd_sim && tr->g_used;
}

// the tile kernels stage the transition in dead scratch (dfx_env_dev.h tile_transition_*): is there enough of it?
static bool transition_fits(const dfx_pack_t* p, int kind, const DfxWalkerParams& w, const DfxPlanarParams& pl, bool backward) {
    if (!p->tile) return false;
    const int no = kind == 1 ? w.num_obs : pl.num_obs, na = kind == 1 ? w.num_act : pl.num_act;
    if (backward) return 2 * no + 3 * (p->header.Q + p->header.D + na) <= p->host.layout_bwd.bwd_size;
    return 2 * no + 1 <= p->host.layout.fwd_size - p->host.layout.act;
}

// the launch-side fields of StepArgs: where the tape's H^-1 blocks start, its dtype, the flags
static void finish_step_args(const dfx_pack_t* p, StepArgs& a) {
    a.hinv_base = tape_geom(p->header.L, p->header.Q, p->header.D, tape_envs(p, a.N), a.substeps, a.mm_freq, p->bf16 != 0).hinv_base;
    a.tape_bf16 = p->bf16;
    a.flags = g_flags;
}

// w: the external wrench (NULL: none -- the kernels without one)
static int run_step(const dfx_pack_t* p, StepArgs& a, bool backward, void* stream, const DfxExternalWrench* w = nullptr) {
    finish_step_args(p, a);
    KernelArgs ka = kernel_args(p, a, w);
    if (p->tile) return counted(tile_api(p->tile)->launch(&ka, backward, w ? 1 : 0, stream));
    cudaStream_t st = (cudaStream_t)stream;
    return w ? run_group<kStepWrench>(p, ka, backward, nullptr, st) : run_group<kStep>(p, ka, backward, nullptr, st);
}

// end state of the recomputed forward: the workspace's tail, q [n*Q] then qd [n*D]
static float* workspace_q_end(const dfx_pack_t* p, const StepArgs& a, float* ws) { return ws + dfx_tape_floats(p, a.N, a.substeps, a.mm_freq); }

// one launch on the tile kernels: the forward into the workspace, the barrier sequence of dfx_tile_recompute_kernel, the adjoint.
// `a` holds the adjoint's arguments (as the stored-tape entry would launch them); the forward's are added here.
static int run_recompute_fused(const dfx_pack_t* p, StepArgs& a, const float* q, const float* qd, float* ws, void* stream,
                               const DfxExternalWrench* w) {
    a.q = q; a.qd = qd;
    a.q_out = workspace_q_end(p, a, ws); a.qd_out = a.q_out + (long long)a.N * p->header.Q;
    a.tape = ws; a.tape_in = ws;
    a.used = nullptr; a.has_derived = 0;
    finish_step_args(p, a);
    KernelArgs ka = kernel_args(p, a, w);
    return counted(tile_api(p->tile)->launch_recompute(&ka, w ? 1 : 0, stream));
}

// the fused kernel exists for every tile pack; the A/B variants of flag bit 6 have none (two launches instead)
static bool recompute_fuses(const dfx_pack_t* p) { return p->tile != 0 && !(g_flags & 64); }

// the recompute adjoint as two launches, where there is no fused kernel: forward(q_end, qd_end) writes the tape into the workspace
// and the end state into its tail, then adjoint() runs the stored-tape entry on it
template <class Forward, class Adjoint>
static int recompute_in_two_launches(const dfx_pack_t* p, const StepArgs& a, float* ws, Forward forward, Adjoint adjoint) {
    float* q_end = workspace_q_end(p, a, ws);
    const int e = forward(q_end, q_end + (long long)a.N * p->header.Q);
    return e != 0 ? e : adjoint();
}

// ---- link state (include/dfx.h dfx_link_state_*): the kernel family the step entries pick for the pack -- its tile kernels, or
// the lane-group kernels of pick_group()'s width, generic under flag bit 2 (4).  The flag-64 A/B variants run the default tile
// kernels (no tape layout to match).
static int run_link_state(const dfx_pack_t* p, int n, const LinkStateArgs& la, bool backward, void* stream) {
    StepArgs a{};
    a.N = n;
    a.flags = g_flags;
    KernelArgs ka = kernel_args(p, a, nullptr);
    if (p->tile) return counted(tile_api(p->tile)->launch_readout(&ka, kReadoutLinkState, &la, backward, stream));
    return run_group<kLinkState>(p, ka, backward, &la, (cudaStream_t)stream);
}

// ---- contact state (include/dfx.h dfx_contact_state_*): on the kernels run_link_state picks
static int run_contact_state(const dfx_pack_t* p, int n, const ContactStateArgs& ca, bool backward, void* stream) {
    StepArgs a{};
    a.N = n;
    a.flags = g_flags;
    KernelArgs ka = kernel_args(p, a, nullptr);
    if (p->tile) return counted(tile_api(p->tile)->launch_readout(&ka, kReadoutContactState, &ca, backward, stream));
    return run_group<kContactState>(p, ka, backward, &ca, (cudaStream_t)stream);
}

// ---- dynamics state (include/dfx.h dfx_dynamics_state_*): on the kernels run_link_state picks.  The backward first runs a
// one-substep env-step (substeps = mm_freq = 1, dt = 0: only its tape row and H^-1 block are used) from the same inputs into the
// workspace, with fp32 rows whatever dfx_set_tape_dtype says -- inside the adjoint's launch on the tile kernels, as the launch
// before on the lane-group kernels -- then the seeded adjoint of its dynamics reads them back.
static TapeGeom dynamics_tape(const dfx_pack_t* p, int n) {
    return tape_geom(p->header.L, p->header.Q, p->header.D, tape_envs(p, n), 1, 1, false);
}

static int run_dynamics_state(const dfx_pack_t* p, int n, const DynamicsStateArgs& da, float* ws, bool backward, void* stream) {
    StepArgs a{};
    a.N = n;
    a.flags = g_flags;
    const DfxExternalWrench w{da.f_ext, nullptr};
    if (backward) {
        const TapeGeom t = dynamics_tape(p, n);
        a.substeps = 1; a.mm_freq = 1;
        a.q = da.q; a.qd = da.qd; a.act = da.act; a.musc = da.musc;
        a.tape = ws; a.tape_in = ws; a.hinv_base = t.hinv_base;
        a.q_out = ws + t.total; a.qd_out = a.q_out + (long long)n * p->header.Q;
    }
    KernelArgs ka = kernel_args(p, a, &w);        // (the tile backward's forward reads ka.wrench; a NULL f_ext is zero)
    if (p->tile) return counted(tile_api(p->tile)->launch_readout(&ka, kReadoutDynamicsState, &da, backward, stream));
    if (backward) {
        const int e = dfx_step_forward_ex(p, n, 1, 1, 0.0, da.q, da.qd, da.act, da.musc, a.q_out, a.qd_out, ws, nullptr, stream,
                                          da.f_ext ? &w : nullptr);
        if (e != 0) return e;
    }
    return run_group<kDynamicsState>(p, ka, backward, &da, (cudaStream_t)stream);
}

// ---- Jacobian state (include/dfx.h dfx_jacobian_state_*): on the kernels run_link_state picks
static int run_jacobian_state(const dfx_pack_t* p, int n, const JacobianStateArgs& ja, bool backward, void* stream) {
    StepArgs a{};
    a.N = n;
    a.flags = g_flags;
    KernelArgs ka = kernel_args(p, a, nullptr);
    if (p->tile) return counted(tile_api(p->tile)->launch_readout(&ka, kReadoutJacobianState, &ja, backward, stream));
    return run_group<kJacobianState>(p, ka, backward, &ja, (cudaStream_t)stream);
}

extern "C" {

int dfx_launch_plan(const dfx_pack_t* p, int backward, int out[6]) {
    if (!p || !out) return (int)cudaErrorInvalidValue;
    const bool bwd = (backward & 1) != 0, wrench = (backward & 2) != 0;
    if (p->tile) {      // one CTA = a tile of E environments
        const KernelArgs ka = kernel_args(p, StepArgs{}, nullptr);
        const size_t smem = tile_api(p->tile)->smem(&ka, backward);
        out[0] = 32; out[1] = p->tile; out[2] = (int)((227 * 1024) / (smem + 1024)); out[3] = (int)smem;
        out[4] = scratch_floats(bwd ? p->host.layout_bwd : p->host.layout, p->header.L, bwd, wrench);
        out[5] = (int)smem - out[4] * p->tile * 4;
        if (wrench && smem > 227 * 1024) out[1] = 0;      // (an articulation whose external-wrench variant no longer fits)
        return 0;
    }
    const int G = pick_group(p);
    const LaunchPlan lp = plan_launch(p, G, bwd, wrench);
    out[0] = G; out[1] = lp.envs_per_cta; out[2] = lp.ctas_per_sm; out[3] = (int)lp.smem;
    out[4] = lp.scratch_stride; out[5] = lp.pack_bytes + lp.cta_area_bytes;
    return 0;
}

int dfx_step_forward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                     const float* q, const float* qd, const float* act, const float* musc,
                     float* q_out, float* qd_out, float* tape, const DfxDerived* derived, void* stream) {
    return dfx_step_forward_ex(p, n, substeps, mm_freq, dt, q, qd, act, musc, q_out, qd_out, tape, derived, stream, nullptr);
}

int dfx_step_forward_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                        const float* q, const float* qd, const float* act, const float* musc,
                        float* q_out, float* qd_out, float* tape, const DfxDerived* derived, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !q || !qd || !act || !q_out || !qd_out || (p->header.M > 0 && !musc))
        return (int)cudaErrorInvalidValue;
    a.q = q; a.qd = qd; a.act = act; a.musc = musc; a.q_out = q_out; a.qd_out = qd_out; a.tape = tape;
    if (derived) { a.derived = *derived; a.has_derived = 1; }
    return run_step(p, a, false, stream, w);
}

int dfx_step_backward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                      const float* act, const float* musc, const float* tape,
                      const float* gq_out, const float* gqd_out,
                      float* gq, float* gqd, float* gact, float* gmusc, void* stream) {
    return dfx_step_backward_ex(p, n, substeps, mm_freq, dt, act, musc, tape, gq_out, gqd_out, gq, gqd, gact, gmusc, stream, nullptr);
}

int dfx_step_backward_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                         const float* act, const float* musc, const float* tape,
                         const float* gq_out, const float* gqd_out,
                         float* gq, float* gqd, float* gact, float* gmusc, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !tape || !act || (p->header.M > 0 && !musc)) return (int)cudaErrorInvalidValue;
    a.act = act; a.musc = musc; a.tape_in = tape; a.gq_out = gq_out; a.gqd_out = gqd_out;
    a.gq = gq; a.gqd = gqd; a.gact = gact; a.gmusc = gmusc;
    return run_step(p, a, true, stream, w);
}

int dfx_step_forward_mapped(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                            const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                            float* used, float* q_out, float* qd_out, float* tape, void* stream) {
    return dfx_step_forward_mapped_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, used, q_out, qd_out, tape, stream, nullptr);
}

int dfx_step_forward_mapped_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                               const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                               float* used, float* q_out, float* qd_out, float* tape, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !q || !qd || !map || !raw || !q_out || !qd_out || !bind_map(p, map, act_other, a))
        return (int)cudaErrorInvalidValue;
    a.q = q; a.qd = qd; a.raw = raw; a.used = used; a.q_out = q_out; a.qd_out = qd_out; a.tape = tape;
    return run_step(p, a, false, stream, w);
}

int dfx_step_backward_mapped(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                             const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                             const float* gq_out, const float* gqd_out, const float* g_used,
                             float* gq, float* gqd, float* g_raw, void* stream) {
    return dfx_step_backward_mapped_ex(p, n, substeps, mm_freq, dt, map, raw, act_other, tape, gq_out, gqd_out, g_used, gq, gqd, g_raw,
                                       stream, nullptr);
}

int dfx_step_backward_mapped_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                                const float* gq_out, const float* gqd_out, const float* g_used,
                                float* gq, float* gqd, float* g_raw, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !tape || !map || !raw || !bind_map(p, map, act_other, a)) return (int)cudaErrorInvalidValue;
    a.raw = raw; a.tape_in = tape; a.gq_out = gq_out; a.gqd_out = gqd_out; a.g_used = g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    return run_step(p, a, true, stream, w);
}

// ---- env.step() as one launch (include/dfx.h): the mapped step with the transition as epilogue (tile kernels), or the two
// launches back to back (lane-group kernels)
int dfx_env_step_forward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                         const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                         float* used, float* q_sim, float* qd_sim, float* tape, const DfxEnvTransition* tr, void* stream) {
    return dfx_env_step_forward_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, used, q_sim, qd_sim, tape, tr, stream, nullptr);
}

int dfx_env_step_forward_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                            const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                            float* used, float* q_sim, float* qd_sim, float* tape, const DfxEnvTransition* tr, void* stream,
                            const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !q || !qd || !map || !raw || !used || !q_sim || !qd_sim || !transition_ok(p, map, tr))
        return (int)cudaErrorInvalidValue;
    if (!transition_fits(p, tr->kind, tr->walker, tr->planar, false)) {
        const int e = dfx_step_forward_mapped_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, used, q_sim, qd_sim, tape, stream, w);
        if (e != 0) return e;
        return tr->kind == 1
            ? dfx_walker_transition_forward(&tr->walker, n, q_sim, qd_sim, used, tr->progress, tr->start_q, tr->start_qd, tr->obs_before, tr->rew,
                                            tr->reset, tr->q_next, tr->qd_next, tr->actions_next, tr->progress_next, tr->obs_next, stream)
            : dfx_planar_transition_forward(&tr->planar, n, q_sim, qd_sim, used, tr->progress, tr->start_q, tr->start_qd, tr->obs_before, tr->rew,
                                            tr->reset, tr->q_next, tr->qd_next, tr->actions_next, tr->progress_next, tr->obs_next, stream);
    }
    if (!bind_map(p, map, act_other, a)) return (int)cudaErrorInvalidValue;
    a.q = q; a.qd = qd; a.raw = raw; a.used = used; a.q_out = q_sim; a.qd_out = qd_sim; a.tape = tape;
    a.env_kind = tr->kind;
    a.env = *tr;
    return run_step(p, a, false, stream, w);
}

int dfx_env_step_backward(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                          const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                          const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream) {
    return dfx_env_step_backward_ex(p, n, substeps, mm_freq, dt, map, raw, act_other, tape, tr, gq, gqd, g_raw, stream, nullptr);
}

int dfx_env_step_backward_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                             const DfxActionMap* map, const float* raw, const float* act_other, const float* tape,
                             const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !tape || !map || !raw || !transition_ok(p, map, tr)) return (int)cudaErrorInvalidValue;
    if (!transition_fits(p, tr->kind, tr->walker, tr->planar, true)) {
        const int e = tr->kind == 1
            ? dfx_walker_transition_backward(&tr->walker, n, tr->q_sim, tr->qd_sim, tr->used, tr->reset, tr->g_obs_before, tr->g_rew, tr->g_q_next,
                                             tr->g_qd_next, tr->g_actions_next, tr->g_obs_next, tr->gq_sim, tr->gqd_sim, tr->g_used, stream)
            : dfx_planar_transition_backward(&tr->planar, n, tr->q_sim, tr->qd_sim, tr->used, tr->reset, tr->g_obs_before, tr->g_rew, tr->g_q_next,
                                             tr->g_qd_next, tr->g_actions_next, tr->g_obs_next, tr->gq_sim, tr->gqd_sim, tr->g_used, stream);
        if (e != 0) return e;
        return dfx_step_backward_mapped_ex(p, n, substeps, mm_freq, dt, map, raw, act_other, tape, tr->gq_sim, tr->gqd_sim, tr->g_used, gq, gqd, g_raw,
                                           stream, w);
    }
    if (!bind_map(p, map, act_other, a)) return (int)cudaErrorInvalidValue;
    a.raw = raw; a.tape_in = tape; a.gq_out = tr->gq_sim; a.gqd_out = tr->gqd_sim; a.g_used = tr->g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    a.env_kind = tr->kind;
    a.env_adj = *tr;
    return run_step(p, a, true, stream, w);
}

// ---- recompute adjoint (include/dfx.h dfx_*_backward_recompute): no stored tape, the env-step's forward is re-run from its
// input state into a one-env-step workspace right before the adjoint reads it
long long dfx_recompute_workspace_floats(const dfx_pack_t* p, int n, int substeps, int mm_freq) {
    if (!p || n <= 0 || substeps <= 0 || mm_freq <= 0) return -1;
    return dfx_tape_floats(p, n, substeps, mm_freq) + (long long)n * (p->header.Q + p->header.D);
}

int dfx_step_backward_recompute(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                const float* q, const float* qd, const float* act, const float* musc, float* workspace,
                                const float* gq_out, const float* gqd_out,
                                float* gq, float* gqd, float* gact, float* gmusc, void* stream) {
    return dfx_step_backward_recompute_ex(p, n, substeps, mm_freq, dt, q, qd, act, musc, workspace, gq_out, gqd_out, gq, gqd, gact, gmusc,
                                          stream, nullptr);
}

int dfx_step_backward_recompute_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                   const float* q, const float* qd, const float* act, const float* musc, float* workspace,
                                   const float* gq_out, const float* gqd_out,
                                   float* gq, float* gqd, float* gact, float* gmusc, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !q || !qd || !workspace || !act || (p->header.M > 0 && !musc))
        return (int)cudaErrorInvalidValue;
    if (!recompute_fuses(p))
        return recompute_in_two_launches(p, a, workspace,
            [&](float* q_end, float* qd_end) {
                return dfx_step_forward_ex(p, n, substeps, mm_freq, dt, q, qd, act, musc, q_end, qd_end, workspace, nullptr, stream, w);
            },
            [&] { return dfx_step_backward_ex(p, n, substeps, mm_freq, dt, act, musc, workspace, gq_out, gqd_out, gq, gqd, gact, gmusc, stream, w); });
    a.act = act; a.musc = musc; a.gq_out = gq_out; a.gqd_out = gqd_out;
    a.gq = gq; a.gqd = gqd; a.gact = gact; a.gmusc = gmusc;
    return run_recompute_fused(p, a, q, qd, workspace, stream, w);
}

int dfx_step_backward_mapped_recompute(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                       const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                       float* workspace, const float* gq_out, const float* gqd_out, const float* g_used,
                                       float* gq, float* gqd, float* g_raw, void* stream) {
    return dfx_step_backward_mapped_recompute_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, workspace, gq_out, gqd_out, g_used,
                                                 gq, gqd, g_raw, stream, nullptr);
}

int dfx_step_backward_mapped_recompute_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                          const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                          float* workspace, const float* gq_out, const float* gqd_out, const float* g_used,
                                          float* gq, float* gqd, float* g_raw, void* stream, const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !q || !qd || !workspace || !map || !raw || !bind_map(p, map, act_other, a))
        return (int)cudaErrorInvalidValue;
    if (!recompute_fuses(p))
        return recompute_in_two_launches(p, a, workspace, 
            [&](float* q_end, float* qd_end) {
                return dfx_step_forward_mapped_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, nullptr, q_end, qd_end, workspace, stream, w);
            },
            [&] {
                return dfx_step_backward_mapped_ex(p, n, substeps, mm_freq, dt, map, raw, act_other, workspace, gq_out, gqd_out, g_used, gq, gqd,
                                                   g_raw, stream, w);
            });
    a.raw = raw; a.gq_out = gq_out; a.gqd_out = gqd_out; a.g_used = g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    return run_recompute_fused(p, a, q, qd, workspace, stream, w);
}

int dfx_env_step_backward_recompute(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                    const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                    float* workspace, const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream) {
    return dfx_env_step_backward_recompute_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, workspace, tr, gq, gqd, g_raw, stream, nullptr);
}

int dfx_env_step_backward_recompute_ex(const dfx_pack_t* p, int n, int substeps, int mm_freq, double dt,
                                       const float* q, const float* qd, const DfxActionMap* map, const float* raw, const float* act_other,
                                       float* workspace, const DfxEnvTransitionAdj* tr, float* gq, float* gqd, float* g_raw, void* stream,
                                       const DfxExternalWrench* w) {
    StepArgs a;
    if (!step_args(p, n, substeps, mm_freq, dt, w, a) || !q || !qd || !workspace || !map || !raw || !transition_ok(p, map, tr) ||
        !bind_map(p, map, act_other, a))
        return (int)cudaErrorInvalidValue;
    // (the stored-tape entry runs the transition adjoint as its prologue or as a launch of its own; the forward needs none of the
    //  transition's outputs: its adjoint reads tr->q_sim, ...)
    if (!recompute_fuses(p) || !transition_fits(p, tr->kind, tr->walker, tr->planar, true))
        return recompute_in_two_launches(p, a, workspace, 
            [&](float* q_end, float* qd_end) {
                return dfx_step_forward_mapped_ex(p, n, substeps, mm_freq, dt, q, qd, map, raw, act_other, nullptr, q_end, qd_end, workspace, stream, w);
            },
            [&] { return dfx_env_step_backward_ex(p, n, substeps, mm_freq, dt, map, raw, act_other, workspace, tr, gq, gqd, g_raw, stream, w); });
    a.raw = raw; a.gq_out = tr->gq_sim; a.gqd_out = tr->gqd_sim; a.g_used = tr->g_used;
    a.gq = gq; a.gqd = gqd; a.g_raw = g_raw;
    a.env_kind = tr->kind;
    a.env_adj = *tr;
    return run_recompute_fused(p, a, q, qd, workspace, stream, w);
}

int dfx_link_state_forward(const dfx_pack_t* p, int n, const float* q, const float* qd,
                           float* body_X_sc, float* body_X_sm, float* body_v_s, void* stream) {
    if (!p || n <= 0 || !q || !qd) return (int)cudaErrorInvalidValue;
    if (!body_X_sc && !body_X_sm && !body_v_s) return 0;
    LinkStateArgs la;
    memset(&la, 0, sizeof la);
    la.q = q; la.qd = qd; la.X_sc = body_X_sc; la.X_sm = body_X_sm; la.v_s = body_v_s;
    return run_link_state(p, n, la, false, stream);
}

int dfx_link_state_backward(const dfx_pack_t* p, int n, const float* q, const float* qd,
                            const float* g_X_sc, const float* g_X_sm, const float* g_v_s,
                            float* gq, float* gqd, void* stream) {
    if (!p || n <= 0 || !q || !qd) return (int)cudaErrorInvalidValue;
    if (!gq && !gqd) return 0;
    LinkStateArgs la;
    memset(&la, 0, sizeof la);
    la.q = q; la.qd = qd; la.g_X_sc = g_X_sc; la.g_X_sm = g_X_sm; la.g_v_s = g_v_s; la.gq = gq; la.gqd = gqd;
    return run_link_state(p, n, la, true, stream);
}

int dfx_contact_state_forward(const dfx_pack_t* p, int n, const float* q, const float* qd,
                              float* contact_f, float* contact_height, float* body_f_contact, void* stream) {
    if (!p || n <= 0 || !q || !qd) return (int)cudaErrorInvalidValue;
    if (!contact_f && !contact_height && !body_f_contact) return 0;
    ContactStateArgs ca;
    memset(&ca, 0, sizeof ca);
    ca.q = q; ca.qd = qd; ca.corder = p->d_corder;
    ca.contact_f = contact_f; ca.contact_height = contact_height; ca.body_f = body_f_contact;
    return run_contact_state(p, n, ca, false, stream);
}

int dfx_contact_state_backward(const dfx_pack_t* p, int n, const float* q, const float* qd,
                               const float* g_contact_f, const float* g_contact_height, const float* g_body_f_contact,
                               float* gq, float* gqd, void* stream) {
    if (!p || n <= 0 || !q || !qd) return (int)cudaErrorInvalidValue;
    if (!gq && !gqd) return 0;
    ContactStateArgs ca;
    memset(&ca, 0, sizeof ca);
    ca.q = q; ca.qd = qd; ca.corder = p->d_corder;
    ca.g_contact_f = g_contact_f; ca.g_contact_height = g_contact_height; ca.g_body_f = g_body_f_contact;
    ca.gq = gq; ca.gqd = gqd;
    return run_contact_state(p, n, ca, true, stream);
}

long long dfx_dynamics_workspace_floats(const dfx_pack_t* p, int n) {
    if (!p || n <= 0) return -1;
    return dynamics_tape(p, n).total + (long long)n * (p->header.Q + p->header.D);
}

int dfx_dynamics_state_forward(const dfx_pack_t* p, int n, const float* q, const float* qd, const float* act, const float* musc,
                               const float* f_ext, float* joint_qdd, float* joint_tau, float* H, void* stream) {
    if (!p || n <= 0 || !q || !qd || !act || (p->header.M > 0 && !musc)) return (int)cudaErrorInvalidValue;
    if (!joint_qdd && !joint_tau && !H) return 0;
    DynamicsStateArgs da;
    memset(&da, 0, sizeof da);
    da.q = q; da.qd = qd; da.act = act; da.musc = musc; da.f_ext = f_ext;
    da.joint_qdd = joint_qdd; da.joint_tau = joint_tau; da.H = H;
    return run_dynamics_state(p, n, da, nullptr, false, stream);
}

int dfx_dynamics_state_backward(const dfx_pack_t* p, int n, const float* q, const float* qd, const float* act, const float* musc,
                                const float* f_ext, float* workspace, const float* g_qdd, const float* g_tau, const float* g_H,
                                float* gq, float* gqd, float* gact, float* gmusc, float* g_f_ext, void* stream) {
    if (!p || n <= 0 || !q || !qd || !act || (p->header.M > 0 && !musc) || !workspace) return (int)cudaErrorInvalidValue;
    if (!gq && !gqd && !gact && !gmusc && !g_f_ext) return 0;
    DynamicsStateArgs da;
    memset(&da, 0, sizeof da);
    da.q = q; da.qd = qd; da.act = act; da.musc = musc; da.f_ext = f_ext;
    da.g_qdd = g_qdd; da.g_tau = g_tau; da.g_H = g_H;
    da.gq = gq; da.gqd = gqd; da.gact = gact; da.gmusc = gmusc; da.g_f_ext = g_f_ext;
    return run_dynamics_state(p, n, da, workspace, true, stream);
}

int dfx_jacobian_state_forward(const dfx_pack_t* p, int n, const float* q, const float* qd, float* J, float* body_a_s, void* stream) {
    if (!p || n <= 0 || !q || !qd) return (int)cudaErrorInvalidValue;
    if (!J && !body_a_s) return 0;
    JacobianStateArgs ja;
    memset(&ja, 0, sizeof ja);
    ja.q = q; ja.qd = qd; ja.J = J; ja.a_s = body_a_s;
    return run_jacobian_state(p, n, ja, false, stream);
}

int dfx_jacobian_state_backward(const dfx_pack_t* p, int n, const float* q, const float* qd, const float* g_J, const float* g_a_s,
                                float* gq, float* gqd, void* stream) {
    if (!p || n <= 0 || !q || !qd) return (int)cudaErrorInvalidValue;
    if (!gq && !gqd) return 0;
    JacobianStateArgs ja;
    memset(&ja, 0, sizeof ja);
    ja.q = q; ja.qd = qd; ja.g_J = g_J; ja.g_a_s = g_a_s; ja.gq = gq; ja.gqd = gqd;
    return run_jacobian_state(p, n, ja, true, stream);
}

}  // extern "C"
