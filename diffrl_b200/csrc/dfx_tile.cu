// dfx_tile.cu -- E-environment tile kernels of the differentiable articulated rigid-body step (sm_90a).
//
// This translation unit is compiled once per tile width:  nvcc -DDFX_TILE_E=E -Ddfx=dfx_eE  with E = 8, 16, 32
// (the namespace is renamed per build so that the three instantiations of the shared headers do not collide).
//
// Execution model: one CTA owns a TILE of E environments for the whole env-step.  A warp holds SUB = 32 / E item slots
// x E environments: lane l of warp w works on item slot  w * SUB + l / E  for environment  l % E  -- the link /
// degree of freedom / contact point / matrix row loops of the phase code (dfx_phases.h `DFX_FOR`) are strided over
// the NW * SUB item slots of the CTA.  E = 32 is the pure "lane = environment, warp = item" mapping of the small
// articulations (Ant, Hopper, HalfCheetah, CartPole); the large ones (Humanoid: 22 links, 16 KB of working set per
// environment; the SNU muscle humanoid) use E = 8 with the compact scratch layouts of dfx_pack.h so that TWO CTAs stay
// resident per SM and hide each other's barrier waits.  Consequences of the mapping:
//   * the per-environment scratch is a structure-of-arrays tile in shared memory (element i of environment e at
//     i * E + e, DFX_ES = E): the E lanes of an item slot hit E consecutive banks, pack reads are broadcasts;
//   * the tape of a tile is [block][tile][row][E]: a substep's rows of the E environments are ONE contiguous block
//     that moves between HBM and the scratch tile as 1-D TMA bulk copies (cp.async.bulk, UBLKCP): one elected thread
//     issues them, loads complete on an mbarrier, stores are fire-and-forget bulk groups -- no thread spends issue
//     slots on moving the tape;
//   * tree recursions cost one item slot per link instead of one (mostly idle) lane group per environment and level;
//   * sparse work (penetrating contact points) is compacted over the whole tile first (cta_compact).
// Every group barrier is a CTA barrier.  The phase code is the same source as the lane-group kernels (dfx_kernels.cu)
// and the host emulation: only the Group policy and the scratch pointer type differ.
#ifndef DFX_TILE_E
#define DFX_TILE_E 32
#endif
#define DFX_ES DFX_TILE_E
#include <cuda_bf16.h>

#include "dfx_launch.h"
#include "dfx_env_dev.h"

namespace dfx {

// ---- 1-D TMA bulk copies and the mbarrier they complete on (PTX: cp.async.bulk, mbarrier)
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "DFX_MBAR_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DFX_MBAR_DONE_%=;\n"
        "bra DFX_MBAR_WAIT_%=;\n"
        "DFX_MBAR_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst_gmem, const void* src_smem, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// make this thread's generic-proxy writes to shared memory visible to the async proxy (before a bulk store reads them)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// every bulk store of this thread has WRITTEN its destination (not only read its source, as bulk_wait_read_all)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// order async-proxy writes to global memory before this thread's later generic-proxy accesses
__device__ __forceinline__ void fence_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

template <int NW, int E, bool PATH>
struct GroupTile {
    static constexpr int SUB = 32 / E;
    static constexpr int G = NW * SUB;           // item slots of the CTA
    static constexpr bool kPathPasses = PATH;    // path / subtree passes instead of per-level tree recursions
#ifndef DFX_TILE_FUSED_PHASES
#define DFX_TILE_FUSED_PHASES 1                  // (0: A/B builds)
#endif
    static constexpr bool kFusedPhases = DFX_TILE_FUSED_PHASES != 0;   // K1 inside integrate_fwd, single-pass tau_adj (dfx_phases.h)
    int lane;            // item slot of DFX_FOR
    int e;               // environment inside the tile
    int tile, ntiles;
    float* tile_base;    // scratch tile (element 0, environment 0)
    int* task_count;
    int* task_list;
    unsigned long long* mbar;      // [2]: head of a tape row (+ H^-1), rest of the row
    mutable unsigned par0, par1;   // their phase parities
    __device__ __forceinline__ void sync() const { __syncthreads(); }
    __device__ __forceinline__ void phase_sync() const {}
    __device__ __forceinline__ void atomic_or(unsigned* p, unsigned v) const { atomicOr(p, v); }
    __device__ __forceinline__ void fx_add(int* p, int v) const { atomicAdd(p, v); }
    __device__ __forceinline__ void atomic_add(float* p, float v) const { atomicAdd(p, v); }
    // max over the item slots of each environment, through the environment's slot
    __device__ __forceinline__ float group_max(float v, SP slot) const {
        if (lane == 0) sp_int(slot)[0] = 0;
        __syncthreads();
        atomicMax(&sp_int(slot)[0], __float_as_int(fmaxf(v, 0.0f)));   // non-negative floats order like ints
        __syncthreads();
        const float m = slot[0];
        __syncthreads();
        return m;
    }
    template <class F>
    __device__ __forceinline__ void cta_tasks(SP s, int n, bool lead, F f) const {
        (void)lead;      // every phase ends with sync(), which is already CTA-wide here
        for (int k = lane; k < n; k += G) f(s, k);
        __syncthreads();
    }
    // append the (k, environment) pairs with pred() true to the CTA-wide list
    template <class Pr>
    __device__ __forceinline__ void compact(SP s, int n, Pr pred) const {
        // (*task_count is 0 on entry: cleared at kernel start and after every use; the preceding phase's closing
        //  barrier has published what pred() reads)
        const int lane32 = threadIdx.x & 31;
        for (int k0 = 0; k0 < n; k0 += G) {
            const int k = k0 + lane;
            const bool hit = (k < n) && pred(s, k);
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (m) {
                int base = 0;
                if (lane32 == 0) base = atomicAdd(task_count, __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (hit) task_list[base + __popc(m & ((1u << lane32) - 1u))] = k * E + e;
            }
        }
        __syncthreads();
    }
    // (k, environment) pairs with pred() true, compacted over the tile, then f() over the list with full warps
    template <class Pr, class F>
    __device__ __forceinline__ void cta_compact(SP s, int n, Pr pred, F f) const {
        compact(s, n, pred);
        const int hits = *task_count;
        for (int i = threadIdx.x; i < hits; i += NW * 32) {
            const int t = task_list[i];
            f(SP{tile_base + (t & (E - 1))}, t / E);
        }
        __syncthreads();
        if (threadIdx.x == 0) *task_count = 0;
    }
    // cta_compact() and m dense items item(s, k) as ONE phase: after the compaction every item slot first does its
    // items, then all warps drain the task list 32 tasks at a time through a shared cursor, so the warps without an
    // item start on the tasks at once and nobody idles while work is left
    static constexpr bool kConcurrentItems = true;
    template <class Pr, class F, class H>
    __device__ __forceinline__ void cta_compact_with(SP s, int n, Pr pred, F f, int m, H item) const {
        int* cursor = task_count + 1;                  // 0 on entry, like *task_count
        compact(s, n, pred);
        const int hits = *task_count;
        for (int k = lane; k < m; k += G) item(s, k);
        const int lane32 = threadIdx.x & 31;
        for (;;) {
            int base = 0;
            if (lane32 == 0) base = atomicAdd(cursor, 32);
            base = __shfl_sync(0xffffffffu, base, 0);
            if (base >= hits) break;
            if (base + lane32 < hits) {
                const int t = task_list[base + lane32];
                f(SP{tile_base + (t & (E - 1))}, t / E);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) { *task_count = 0; *cursor = 0; }
    }

    // ---- tape blocks [b][tile][n][E]: the scratch tile of the block is the same bytes.
    // Stores: every thread fences its scratch writes towards the async proxy, the CTA meets, one thread issues the
    // bulk copy as its own bulk group.  The source must stay untouched until the copy has READ it: row_reusable() /
    // finish() below.
    __device__ __forceinline__ void block_out(float* base, long long b, int N, int env, SP src, int n, bool rows) const {
        (void)N; (void)env; (void)rows;
        fence_async_smem();
        __syncthreads();
        if (threadIdx.x == 0) {
            bulk_store(base + ((b * ntiles + tile) * n) * E, sp_raw(src) - e, (unsigned)(n * E * 4));
            bulk_commit();
        }
    }
    // a tape row as bulk stores: (q, qd) when the substep starts; the intermediates and q'' when they exist.  With a bf16
    // tape the middle is first converted into the staging area (flat: the tile's [head, tail) x E floats are contiguous).
    // `fenced`: every thread called pre_store() before the CTA's last barrier and nothing the store reads was written since
    __device__ __forceinline__ void block_out_part(float* base, long long b, int N, int env, SP src, const RowFmt& f, SP stage, bool first, bool fenced = false) const {
        (void)N; (void)env;
        float* sm = sp_raw(src) - e;
        float* st = sp_raw(stage) - e;
        if (!first && f.bf16) {
            const float2* in = reinterpret_cast<const float2*>(sm + f.head * E);
            __nv_bfloat162* out = reinterpret_cast<__nv_bfloat162*>(st);
            for (int i = threadIdx.x; i < (f.tail - f.head) * E / 2; i += NW * 32) out[i] = __float22bfloat162_rn(in[i]);
        }
        if (!fenced) {
            fence_async_smem();
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            float* d = base + ((b * ntiles + tile) * f.units) * E;
            if (first) {
                bulk_store(d, sm, (unsigned)(f.early * E * 4));
            } else if (!f.bf16) {
                bulk_store(d + f.early * E, sm + f.early * E, (unsigned)((f.n - f.early) * E * 4));
            } else {
                const int mid_units = (f.tail - f.head) / 2;
                bulk_store(d + f.early * E, sm + f.early * E, (unsigned)((f.head - f.early) * E * 4));     // link transforms + S, fp32
                bulk_store(d + f.head * E, st, (unsigned)(mid_units * E * 4));                               // v, a, f_tot as bf16
                bulk_store(d + (f.head + mid_units) * E, sm + f.tail * E, (unsigned)((f.n - f.tail) * E * 4));
            }
            bulk_commit();
        }
    }
    __device__ __forceinline__ void pre_store() const { fence_async_smem(); }
    __device__ __forceinline__ void store_sync() const {}
    // called before the first barrier after which the scratch row (and H^-1) may be overwritten again
    __device__ __forceinline__ void row_reusable() const { if (threadIdx.x == 0) bulk_wait_read_all(); }
    __device__ __forceinline__ void finish() const { if (threadIdx.x == 0) bulk_wait_read_all(); }

    // Loads (adjoint): a row arrives in two parts, each completing on its own mbarrier: first the element ranges
    // [0, head) and [tail, n) -- (q, qd) and q'', all that the first two adjoint phases read -- together with the H^-1
    // block when `hinv_dst` is given, then the middle [head, tail).  The caller's preceding CTA barrier guarantees
    // that nobody still reads the destinations.
    __device__ __forceinline__ void row_in(SP dst, const float* base, long long b, int N, int env, int n, int head, int tail, bool first) const {
        (void)N; (void)env; (void)dst; (void)base; (void)b; (void)n; (void)head; (void)tail; (void)first;   // (see rows_in)
    }
    __device__ __forceinline__ void rows_in(SP dst, const float* base, long long b, const RowFmt& f, SP stage,
                                            SP hinv_dst, const float* hinv_src, int dd) const {
        if (threadIdx.x != 0) return;
        const float* src = base + ((b * ntiles + tile) * f.units) * E;
        float* d = sp_raw(dst) - e;
        const int mid_units = f.bf16 ? (f.tail - f.head) / 2 : (f.tail - f.head);
        const unsigned b_early = (unsigned)(f.early * E * 4), b_tail = (unsigned)((f.n - f.tail) * E * 4);
        const unsigned b_xf = (unsigned)((f.head - f.early) * E * 4), b_mid = (unsigned)(mid_units * E * 4);
        const unsigned b_hinv = hinv_src ? (unsigned)(dd * E * 4) : 0u;
        mbar_arrive_expect_tx(&mbar[0], b_early + b_tail + b_hinv);
        bulk_load(d, src, b_early, &mbar[0]);
        if (b_tail) bulk_load(d + f.tail * E, src + (f.head + mid_units) * E, b_tail, &mbar[0]);
        if (b_hinv) bulk_load(sp_raw(hinv_dst) - e, hinv_src, b_hinv, &mbar[0]);
        mbar_arrive_expect_tx(&mbar[1], b_xf + b_mid);
        if (b_xf) bulk_load(d + f.early * E, src + f.early * E, b_xf, &mbar[1]);
        bulk_load(f.bf16 ? sp_raw(stage) - e : d + f.head * E, src + f.head * E, b_mid, &mbar[1]);
    }
    // pull the row the NEXT iteration will load (the previous substep's) into L2 while this substep's adjoint runs: its
    // bulk loads then complete from L2 instead of paying the HBM latency at the top of every substep
    __device__ __forceinline__ void prefetch_row(const float* base, long long b, const RowFmt& f) const {
        if (threadIdx.x != 0) return;
        const float* src = base + ((b * ntiles + tile) * f.units) * E;
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"((unsigned)(f.units * E * 4)) : "memory");
    }
    // bf16 tape: after copy_wait_all() the staged halves are widened into the scratch fields [head, tail)
    __device__ __forceinline__ void row_unpack(SP dst, SP stage, const RowFmt& f) const {
        if (!f.bf16) return;
        const __nv_bfloat162* in = reinterpret_cast<const __nv_bfloat162*>(sp_raw(stage) - e);
        float2* out = reinterpret_cast<float2*>(sp_raw(dst) - e + f.head * E);
        for (int i = threadIdx.x; i < (f.tail - f.head) * E / 2; i += NW * 32) out[i] = __bfloat1622float2(in[i]);
    }
    __device__ __forceinline__ const float* block_ptr(const float* base, long long b, int n) const { return base + ((b * ntiles + tile) * n) * E; }
    __device__ __forceinline__ void block_in(SP dst, const float* base, long long b, int N, int env, int n, bool rows) const {
        (void)dst; (void)base; (void)b; (void)N; (void)env; (void)n; (void)rows;      // (folded into rows_in)
    }
    __device__ __forceinline__ HinvView hinv_view(const float* base, long long b, int N, int env, int n) const {
        (void)N; (void)env;
        return HinvView{base + ((b * ntiles + tile) * n) * E + e, E};
    }
    __device__ __forceinline__ void copy_wait_first() const { mbar_wait(&mbar[0], par0); par0 ^= 1u; }
    __device__ __forceinline__ void copy_wait_all() const { mbar_wait(&mbar[1], par1); par1 ^= 1u; }
    static constexpr bool kBulkRows = true;     // env_step_backward uses rows_in()
};

template <int NW, int MINB, bool BACKWARD, bool PATH, int MODE, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(NW * 32, MINB) dfx_tile_kernel(const __grid_constant__ KernelArgs ka) {
    constexpr int E = DFX_TILE_E;
    extern __shared__ __align__(128) float smem[];
    float* fpack = smem;
    int* ipack = reinterpret_cast<int*>(smem + ((ka.blob.n_floats + 3) & ~3));
    for (int i = threadIdx.x; i < ka.blob.n_floats; i += NW * 32) fpack[i] = ka.blob.floats[i];
    for (int i = threadIdx.x; i < ka.blob.n_ints; i += NW * 32) ipack[i] = ka.blob.ints[i];
    int* cta_area = reinterpret_cast<int*>(smem + ka.pack_smem_floats);
    if (threadIdx.x < 4) cta_area[threadIdx.x] = 0;   // task counter / cursor of cta_compact
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(cta_area + 4);
    if (threadIdx.x == 0) {
        mbar_init(&mbar[0], 1);
        mbar_init(&mbar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    Pack P = bind_pack(ka.header, ka.blob, ipack, fpack);
    P.L = SL; P.D = SD; P.Q = SQ; P.C = SC; P.M = SM;
    P.jmask = tile_joint_mask(SL, SD, SQ, SC, SM);      // (dfx_pack_create checked that the links have no other joint type)
    constexpr Layout Y = make_layout(SL, SD, SQ, SC, SM, MODE, BACKWARD);

    GroupTile<NW, E, PATH> g;
    const int lane32 = threadIdx.x & 31;
    g.lane = (threadIdx.x >> 5) * (32 / E) + lane32 / E;
    g.e = lane32 % E;
    g.tile = blockIdx.x;
    g.ntiles = gridDim.x;
    g.task_count = cta_area;
    g.task_list = cta_area + 8;
    g.mbar = mbar;
    g.par0 = g.par1 = 0u;
    g.tile_base = smem + ka.pack_smem_floats + ka.cta_area_floats;
    // lanes past the end redo the last environment: identical values are stored twice, every thread reaches
    // every barrier, and the (padded) tape tile slots of those lanes are simply never read by anybody else
    int env = blockIdx.x * E + g.e;
    if (env >= ka.step.N) env = ka.step.N - 1;
    const SP s{g.tile_base + g.e};
    // env.step() as one launch (dfx_env_step_forward / _backward): the transition of this tile's environments -- observation,
    // reward, termination, masked re-initialisation, next observation -- runs as the epilogue of the simulation step, its adjoint
    // as the prologue of the step adjoint, both staged in the scratch tile (dfx_env_dev.h tile_transition_*): thread e < E
    // evaluates environment e in shared memory, all threads move the rows.  The cotangents of (q_sim, qd_sim, used) reach the step
    // adjoint through three small global work arrays written and read by this CTA only, on either side of a CTA barrier.
    if (BACKWARD) {
        if (ka.step.env_kind) tile_transition_backward<NW * 32, E>(ka.step.env_kind, ka.step.env_adj, g.tile_base, ka.step.N);
        env_step_backward(P, Y, s, g, env, ka.step);
    } else {
        env_step_forward(P, Y, s, g, env, ka.step);
        if (ka.step.env_kind) {
            // the stepped state is still in the scratch tile; everything past the tape row (actuation, tau, H^-1, ...) is dead:
            // that is where the observations are formed.  `used` (global) was written by this CTA before the barrier.
            g.row_reusable();           // (no bulk store -- the H^-1 block of a last-substep update -- still reads that region)
            __syncthreads();
            tile_transition_forward<NW * 32, E>(ka.step.env_kind, ka.step.env, ka.step.used, g.tile_base, Y.q, Y.qd, Y.act, ka.step.N);
        }
    }
    g.finish();
}

// Recompute adjoint (include/dfx.h dfx_*_backward_recompute): the env-step's forward, re-run from its input state, writes the
// tape of this tile into a caller-supplied one-env-step workspace (ka.step.tape, the tape's own layout) and the end state to
// ka.step.q_out / qd_out (its tail); then the adjoint of dfx_tile_kernel<BACKWARD = true> reads that tape back
// (ka.step.tape_in == ka.step.tape).  The forward is deterministic -- fixed-point scatter-adds, no float atomics -- so the
// recomputed rows and H^-1 blocks are the stored tape's bit for bit.  Same set-up as dfx_tile_kernel (which stays as it is),
// scratch sized for the larger of the two layouts, the backward's warps and occupancy.
template <int NW, int MINB, bool PATH, int MODE, int SL, int SD, int SQ, int SC, int SM>
__global__ void __launch_bounds__(NW * 32, MINB) dfx_tile_recompute_kernel(const __grid_constant__ KernelArgs ka) {
    constexpr int E = DFX_TILE_E;
    extern __shared__ __align__(128) float smem[];
    float* fpack = smem;
    int* ipack = reinterpret_cast<int*>(smem + ((ka.blob.n_floats + 3) & ~3));
    for (int i = threadIdx.x; i < ka.blob.n_floats; i += NW * 32) fpack[i] = ka.blob.floats[i];
    for (int i = threadIdx.x; i < ka.blob.n_ints; i += NW * 32) ipack[i] = ka.blob.ints[i];
    int* cta_area = reinterpret_cast<int*>(smem + ka.pack_smem_floats);
    if (threadIdx.x < 4) cta_area[threadIdx.x] = 0;
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(cta_area + 4);
    if (threadIdx.x == 0) {
        mbar_init(&mbar[0], 1);
        mbar_init(&mbar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    Pack P = bind_pack(ka.header, ka.blob, ipack, fpack);
    P.L = SL; P.D = SD; P.Q = SQ; P.C = SC; P.M = SM;
    P.jmask = tile_joint_mask(SL, SD, SQ, SC, SM);
    constexpr Layout YF = make_layout(SL, SD, SQ, SC, SM, MODE, false);
    constexpr Layout YB = make_layout(SL, SD, SQ, SC, SM, MODE, true);

    GroupTile<NW, E, PATH> g;
    const int lane32 = threadIdx.x & 31;
    g.lane = (threadIdx.x >> 5) * (32 / E) + lane32 / E;
    g.e = lane32 % E;
    g.tile = blockIdx.x;
    g.ntiles = gridDim.x;
    g.task_count = cta_area;
    g.task_list = cta_area + 8;
    g.mbar = mbar;
    g.par0 = g.par1 = 0u;
    g.tile_base = smem + ka.pack_smem_floats + ka.cta_area_floats;
    int env = blockIdx.x * E + g.e;
    if (env >= ka.step.N) env = ka.step.N - 1;
    const SP s{g.tile_base + g.e};

    env_step_forward(P, YF, s, g, env, ka.step);     // (no `used`, no derived dumps, no transition epilogue)
    // The adjoint below reads the workspace the forward's bulk stores are still writing: TMA bulk loads of the rows (issued by
    // thread 0) and, in the layouts without a staged H^-1 (Y.A < 0: the humanoids), plain loads of H^-1 rows by every thread.
    //  1. every thread: fence its generic writes to the scratch tile against the async proxy -- the adjoint's bulk loads
    //     overwrite the same bytes;
    //  2. thread 0, the only issuer of bulk stores: wait_group 0 waits until they have WRITTEN global memory (wait_group.read,
    //     all the forward needs, only waits until they have read the scratch), then a proxy fence orders those async-proxy
    //     writes before generic-proxy accesses;
    //  3. the CTA barrier publishes 1. and 2. to every thread: a bulk load issued or a plain load executed after it sees the
    //     tape rows and H^-1 blocks the forward wrote.  Each CTA reads only its own tile's slots, so no other CTA is involved.
    fence_async_smem();
    if (threadIdx.x == 0) {
        bulk_wait_all();
        fence_async_global();
    }
    __syncthreads();
    if (ka.step.env_kind) tile_transition_backward<NW * 32, E>(ka.step.env_kind, ka.step.env_adj, g.tile_base, ka.step.N);
    env_step_backward(P, YB, s, g, env, ka.step);
    g.finish();
}

// 128-byte aligned offsets so that the bulk copies of the tile stay 16-byte aligned
static int tile_pack_floats(const KernelArgs& ka) {
    const int bytes = (((ka.blob.n_floats + 3) & ~3) + ((ka.blob.n_ints + 3) & ~3)) * 4;
    return ((bytes + 127) & ~127) / 4;
}
// CTA area: 4 ints (task counter, cursor), 2 mbarriers (16 bytes), then one list slot per (contact point, environment)
static int tile_area_floats(const KernelArgs& ka) { return ((32 + ka.header.C * DFX_TILE_E * 4 + 127) & ~127) / 4; }

template <int NW, int MINB, bool BWD, bool PATH, int MODE, int SL, int SD, int SQ, int SC, int SM>
static cudaError_t tile_launch_impl(KernelArgs& ka, cudaStream_t stream) {
    constexpr Layout Y = make_layout(SL, SD, SQ, SC, SM, MODE, BWD);
    const int per_env = ((BWD ? Y.bwd_size : Y.fwd_size) + 3) & ~3;
    ka.layout = Y;
    ka.pack_smem_floats = tile_pack_floats(ka);
    ka.cta_area_floats = tile_area_floats(ka);
    ka.scratch_stride = per_env;
    const size_t smem = (size_t)(ka.pack_smem_floats + ka.cta_area_floats + per_env * DFX_TILE_E) * sizeof(float);
    auto kern = dfx_tile_kernel<NW, MINB, BWD, PATH, MODE, SL, SD, SQ, SC, SM>;
    // (the opt-in to > 48 KB of dynamic shared memory is per device: set it on every launch, it is cheap)
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int ntiles = (ka.step.N + DFX_TILE_E - 1) / DFX_TILE_E;
    kern<<<ntiles, NW * 32, smem, stream>>>(ka);
    return cudaGetLastError();
}

template <int NW, int MINB, bool PATH, int MODE, int SL, int SD, int SQ, int SC, int SM>
static cudaError_t tile_recompute_launch_impl(KernelArgs& ka, cudaStream_t stream) {
    constexpr Layout YF = make_layout(SL, SD, SQ, SC, SM, MODE, false);
    constexpr Layout YB = make_layout(SL, SD, SQ, SC, SM, MODE, true);
    const int per_env = ((YF.fwd_size > YB.bwd_size ? YF.fwd_size : YB.bwd_size) + 3) & ~3;
    ka.layout = YB;
    ka.pack_smem_floats = tile_pack_floats(ka);
    ka.cta_area_floats = tile_area_floats(ka);
    ka.scratch_stride = per_env;
    const size_t smem = (size_t)(ka.pack_smem_floats + ka.cta_area_floats + per_env * DFX_TILE_E) * sizeof(float);
    auto kern = dfx_tile_recompute_kernel<NW, MINB, PATH, MODE, SL, SD, SQ, SC, SM>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int ntiles = (ka.step.N + DFX_TILE_E - 1) / DFX_TILE_E;
    kern<<<ntiles, NW * 32, smem, stream>>>(ka);
    return cudaGetLastError();
}

}  // namespace dfx

using namespace dfx;

// The articulations with a tile kernel of this width:
//   X(warps forward, warps backward, min CTAs per SM (register budget), path passes, layout mode, L, D, Q, C, M)
#ifndef DFX_TILE_NWF         // warps of the Ant tile kernels (tuning builds: -DDFX_TILE_NWF=12 -DDFX_TILE_NWB=12 -DDFX_TILE_ONLY_ANT)
#define DFX_TILE_NWF 16
#endif
#ifndef DFX_TILE_NWB
#define DFX_TILE_NWB 16
#endif
#if DFX_TILE_E == 32
#ifdef DFX_TILE_ONLY_ANT      // (tuning builds)
#define DFX_TILE_MODELS(X) X(DFX_TILE_NWF, DFX_TILE_NWB, 1, true, 0, 9, 14, 15, 25, 0)
#else
#define DFX_TILE_MODELS(X)                                        \
    X(DFX_TILE_NWF, DFX_TILE_NWB, 1, true, 0, 9, 14, 15, 25, 0) /* Ant */             \
    X(8, 8, 1, true, 0, 3, 2, 2, 0, 0)      /* CartPole */        \
    X(16, 16, 1, true, 0, 6, 6, 6, 8, 0)    /* Hopper */          \
    X(16, 16, 1, true, 0, 9, 9, 9, 16, 0)   /* HalfCheetah */
#endif
#elif DFX_TILE_E == 16
#define DFX_TILE_MODELS(X)                                        \
    X(8, 8, 2, true, 3 | 16, 9, 14, 15, 25, 0)   /* Ant, two CTAs per SM (A/B only) */   \
    X(16, 16, 1, true, 3 | 16, 22, 27, 28, 35, 0) /* Humanoid, one CTA of 16 environments per SM (A/B only: 8 x 2 CTAs is 1-4 % faster) */ \
    X(16, 16, 1, true, 3, 11, 24, 29, 88, 152)    /* SNU humanoid: one CTA of 16 environments, 16 warps (7 % faster than 8 x 2 CTAs: 152 muscles fill the slots) */
#elif DFX_TILE_E == 8
#define DFX_TILE_MODELS(X)                                        \
    X(8, 8, 2, true, 3, 22, 27, 28, 35, 0)    /* Humanoid */      \
    X(8, 8, 2, true, 3 | 16, 11, 24, 29, 88, 152)  /* SNU humanoid (A/B only: its default is E = 16) */ \
    X(4, 4, 4, true, 3 | 16, 9, 14, 15, 25, 0)     /* Ant, four CTAs per SM (A/B only) */
#endif

// alternative instantiations, picked by flag bit 6 (64) of dfx_set_flags (A/B timing): level-by-level tree recursions
#if DFX_TILE_E == 8
#define DFX_TILE_MODELS_ALT(X)                                    \
    X(8, 8, 2, false, 3, 22, 27, 28, 35, 0)    /* Humanoid */     \
    X(8, 8, 2, false, 3, 11, 24, 29, 88, 152)  /* SNU humanoid */
#else
#define DFX_TILE_MODELS_ALT(X)
#endif

#define DFX_CAT2(a, b) a##b
#define DFX_CAT(a, b) DFX_CAT2(a, b)
#define DFX_TILE_FN(name) DFX_CAT(DFX_CAT(name, _e), DFX_TILE_E)

// layout mode of the tile kernel for this articulation (bit 4 (16): instantiated for A/B runs only, never picked
// automatically), or -1 when there is none of this width
int DFX_TILE_FN(dfx_tile_mode)(int L, int D, int Q, int C, int M) {
#define X(nwf, nwb, minb, path, mode, l, d, q, c, m) if (L == l && D == d && Q == q && C == c && M == m) return mode;
    DFX_TILE_MODELS(X)
#undef X
    return -1;
}

// dynamic shared memory of the tile kernel (bytes): pack + CTA area + E x scratch
size_t DFX_TILE_FN(dfx_tile_smem)(const void* kargs, int backward) {
    const KernelArgs& ka = *static_cast<const KernelArgs*>(kargs);
    const int mode = DFX_TILE_FN(dfx_tile_mode)(ka.header.L, ka.header.D, ka.header.Q, ka.header.C, ka.header.M);
    const Layout Y = make_layout(ka.header.L, ka.header.D, ka.header.Q, ka.header.C, ka.header.M, mode < 0 ? 0 : (mode & 3), backward != 0);
    const int per_env = ((backward ? Y.bwd_size : Y.fwd_size) + 3) & ~3;
    return (size_t)(tile_pack_floats(ka) + tile_area_floats(ka) + per_env * DFX_TILE_E) * sizeof(float);
}

int DFX_TILE_FN(dfx_tile_launch)(void* kargs, int backward, void* stream) {
    KernelArgs& ka = *static_cast<KernelArgs*>(kargs);
    const Pack& h = ka.header;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
#define X(nwf, nwb, minb, path, mode, l, d, q, c, m)                                                   \
    if (h.L == l && h.D == d && h.Q == q && h.C == c && h.M == m)                                      \
        return (int)(backward ? tile_launch_impl<nwb, minb, true, path, (mode) & 3, l, d, q, c, m>(ka, st)   \
                              : tile_launch_impl<nwf, minb, false, path, (mode) & 3, l, d, q, c, m>(ka, st));
    if (ka.step.flags & 64) { DFX_TILE_MODELS_ALT(X) }
    DFX_TILE_MODELS(X)
#undef X
    return (int)cudaErrorInvalidConfiguration;
}

// the recompute adjoint (dfx_tile_recompute_kernel) of every DFX_TILE_MODELS entry, with the backward kernel's warps and
// occupancy (every entry has as many forward as backward warps; tuning builds that set them apart run the forward part with
// the backward's).  No flag-64 (A/B) variants: the caller runs the forward and the backward launches instead.
int DFX_TILE_FN(dfx_tile_launch_recompute)(void* kargs, void* stream) {
    KernelArgs& ka = *static_cast<KernelArgs*>(kargs);
    const Pack& h = ka.header;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
#define X(nwf, nwb, minb, path, mode, l, d, q, c, m)                                                   \
    if (h.L == l && h.D == d && h.Q == q && h.C == c && h.M == m)                                      \
        return (int)tile_recompute_launch_impl<nwb, minb, path, (mode) & 3, l, d, q, c, m>(ka, st);
    DFX_TILE_MODELS(X)
#undef X
    return (int)cudaErrorInvalidConfiguration;
}
