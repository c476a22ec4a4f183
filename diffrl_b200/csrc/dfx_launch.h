// dfx_launch.h -- launch-side structs shared by the lane-group kernels (dfx_kernels.cu) and the 32-environment
// tile kernels (dfx_tile.cu): the packed model blob, its staging into shared memory, the kernel argument block.
#pragma once

#include <cuda_runtime.h>

#include "dfx_step.h"

namespace dfx {

constexpr int kMaxThreads = 128;

// Copy the pack's arrays into shared memory once per CTA and rebind the pointers.
struct PackBlob {
    const int* ints;
    const float* floats;
    int n_ints, n_floats;
    // offsets of each pointer field (same order as PackHost::bind)
    int int_off[26];
    int float_off[17];
};

__device__ __forceinline__ Pack bind_pack(const Pack& header, const PackBlob& b, const int* ib, const float* fb) {
    Pack p = header;
    int ii = 0, fi = 0;
    p.type = ib + b.int_off[ii++]; p.parent = ib + b.int_off[ii++]; p.q_start = ib + b.int_off[ii++];
    p.qd_start = ib + b.int_off[ii++]; p.level_start = ib + b.int_off[ii++]; p.level_links = ib + b.int_off[ii++];
    p.child_start = ib + b.int_off[ii++]; p.child_idx = ib + b.int_off[ii++]; p.anc_start = ib + b.int_off[ii++];
    p.anc_dofs = ib + b.int_off[ii++]; p.sub_start = ib + b.int_off[ii++]; p.sub_links = ib + b.int_off[ii++];
    p.path_start = ib + b.int_off[ii++]; p.path_links = ib + b.int_off[ii++]; p.round_start = ib + b.int_off[ii++];
    p.chain_start = ib + b.int_off[ii++]; p.chain_links = ib + b.int_off[ii++];
    p.dof_link = ib + b.int_off[ii++]; p.cbody_start = ib + b.int_off[ii++]; p.cbody = ib + b.int_off[ii++];
    p.mstart = ib + b.int_off[ii++]; p.mlinks = ib + b.int_off[ii++];
    p.aseg_start = ib + b.int_off[ii++]; p.aseg_way = ib + b.int_off[ii++]; p.morder = ib + b.int_off[ii++]; p.mgrp_start = ib + b.int_off[ii++];
    p.X_pj = fb + b.float_off[fi++]; p.X_cm = fb + b.float_off[fi++]; p.axis = fb + b.float_off[fi++];
    p.I_c = fb + b.float_off[fi++]; p.mass = fb + b.float_off[fi++]; p.target_ke = fb + b.float_off[fi++];
    p.target_kd = fb + b.float_off[fi++]; p.limit_ke = fb + b.float_off[fi++]; p.limit_kd = fb + b.float_off[fi++];
    p.target = fb + b.float_off[fi++]; p.limit_lower = fb + b.float_off[fi++]; p.limit_upper = fb + b.float_off[fi++];
    p.armature = fb + b.float_off[fi++]; p.cpoint = fb + b.float_off[fi++]; p.cdist = fb + b.float_off[fi++];
    p.cmat = fb + b.float_off[fi++]; p.mpoints = fb + b.float_off[fi++];
    return p;
}

// joint types the size-specialised tile kernel of an articulation is COMPILED for (Pack::jmask as a constant: the branches of
// the other types are not in the binary).  A pack whose links have any other type never gets a tile kernel (dfx_pack_create falls
// back to the lane-group kernels, which read the mask at run time).
DFX_LAYOUT_FN int tile_joint_mask(int L, int D, int Q, int C, int M) {
    constexpr int P = 1 << JOINT_PRISMATIC, R = 1 << JOINT_REVOLUTE, B = 1 << JOINT_BALL, F = 1 << JOINT_FREE;
    if (L == 9 && D == 14 && Q == 15 && C == 25 && M == 0) return F | R;          // Ant
    if (L == 22 && D == 27 && Q == 28 && C == 35 && M == 0) return F | R;         // Humanoid
    if (L == 11 && D == 24 && Q == 29 && C == 88 && M == 152) return F | B | R;   // SNU humanoid
    if (L == 3 && D == 2 && Q == 2 && C == 0 && M == 0) return P | R | (1 << JOINT_FIXED);   // CartPole (fixed rail link)
    if (L == 6 && D == 6 && Q == 6 && C == 8 && M == 0) return P | R;             // Hopper
    if (L == 9 && D == 9 && Q == 9 && C == 16 && M == 0) return P | R;            // HalfCheetah
    return kJointMaskAll;
}

struct KernelArgs {
    Pack header;
    PackBlob blob;
    Layout layout;
    StepArgs step;
    int scratch_stride;   // floats per environment
    int pack_smem_floats; // floats reserved at the start of dynamic smem for the staged pack
    int cta_area_floats;  // then: CTA-wide task counter + task list (cta_compact)
};


}  // namespace dfx

// ---- tile kernels (dfx_tile.cu, compiled once per tile width E = 8, 16, 32 with its own namespace): one CTA = E
// environments.  KernelArgs is a plain struct with the same layout in every build; it crosses as void*.
#define DFX_DECLARE_TILE(E)                                                                                           \
    int dfx_tile_mode_e##E(int L, int D, int Q, int C, int M);      /* layout mode, or -1: no kernel of this width */  \
    size_t dfx_tile_smem_e##E(const void* kernel_args, int backward); /* dynamic shared memory (bytes) */             \
    int dfx_tile_launch_e##E(void* kernel_args, int backward, void* stream);                                         \
    int dfx_tile_launch_recompute_e##E(void* kernel_args, void* stream);   /* forward into the workspace + adjoint, one launch */
DFX_DECLARE_TILE(8)
DFX_DECLARE_TILE(16)
DFX_DECLARE_TILE(32)
#undef DFX_DECLARE_TILE
