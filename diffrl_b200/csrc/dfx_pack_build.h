// dfx_pack_build.h -- host-side construction of the ModelPack from a DfxModelDesc:
// validation, tree levels, children / ancestor-dof / subtree lists, contact grouping by body.
// Produces two flat host arrays (ints, floats) and the offsets of every Pack field in them, so
// the same builder serves the CUDA library (arrays copied to the device) and the host
// emulation harness used by the CPU-side unit tests.
#pragma once

#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/dfx.h"
#include "dfx_pack.h"

namespace dfx {

struct PackHost {
    std::vector<int> ints;
    std::vector<float> floats;
    // offsets into ints / floats, in the order of the pointer fields of Pack
    std::vector<size_t> int_off, float_off;
    Pack header;  // scalar fields filled; pointer fields filled by bind()
    std::vector<int> corder;   // (C) Model index of the pack's contact n (not staged: read by the contact state only)
    Layout layout;       // forward kernels (legacy mode: also the backward kernels)
    Layout layout_bwd;   // backward kernels
    int layout_mode = kLayoutLegacy;
    void set_layout_mode(int mode) {
        layout_mode = mode;
        layout = make_layout(header.L, header.D, header.Q, header.C, header.M, mode, false);
        layout_bwd = make_layout(header.L, header.D, header.Q, header.C, header.M, mode, true);
    }

    // point the Pack's pointer fields at (ibase, fbase)
    Pack bind(const int* ibase, const float* fbase) const {
        Pack p = header;
        size_t ii = 0, fi = 0;
        p.type = ibase + int_off[ii++];
        p.parent = ibase + int_off[ii++];
        p.q_start = ibase + int_off[ii++];
        p.qd_start = ibase + int_off[ii++];
        p.level_start = ibase + int_off[ii++];
        p.level_links = ibase + int_off[ii++];
        p.child_start = ibase + int_off[ii++];
        p.child_idx = ibase + int_off[ii++];
        p.anc_start = ibase + int_off[ii++];
        p.anc_dofs = ibase + int_off[ii++];
        p.sub_start = ibase + int_off[ii++];
        p.sub_links = ibase + int_off[ii++];
        p.path_start = ibase + int_off[ii++];
        p.path_links = ibase + int_off[ii++];
        p.round_start = ibase + int_off[ii++];
        p.chain_start = ibase + int_off[ii++];
        p.chain_links = ibase + int_off[ii++];
        p.dof_link = ibase + int_off[ii++];
        p.cbody_start = ibase + int_off[ii++];
        p.cbody = ibase + int_off[ii++];
        p.mstart = ibase + int_off[ii++];
        p.mlinks = ibase + int_off[ii++];
        p.aseg_start = ibase + int_off[ii++];
        p.aseg_way = ibase + int_off[ii++];
        p.morder = ibase + int_off[ii++];
        p.mgrp_start = ibase + int_off[ii++];
        p.X_pj = fbase + float_off[fi++];
        p.X_cm = fbase + float_off[fi++];
        p.axis = fbase + float_off[fi++];
        p.I_c = fbase + float_off[fi++];
        p.mass = fbase + float_off[fi++];
        p.target_ke = fbase + float_off[fi++];
        p.target_kd = fbase + float_off[fi++];
        p.limit_ke = fbase + float_off[fi++];
        p.limit_kd = fbase + float_off[fi++];
        p.target = fbase + float_off[fi++];
        p.limit_lower = fbase + float_off[fi++];
        p.limit_upper = fbase + float_off[fi++];
        p.armature = fbase + float_off[fi++];
        p.cpoint = fbase + float_off[fi++];
        p.cdist = fbase + float_off[fi++];
        p.cmat = fbase + float_off[fi++];
        p.mpoints = fbase + float_off[fi++];
        return p;
    }
};

inline bool build_pack(const DfxModelDesc& d, PackHost& out, std::string& err) {
    const int L = d.link_count, D = d.dof_count, Q = d.coord_count, C = d.contact_count;
    const int M = d.muscle_count, W = d.waypoint_count;
    char buf[256];
    if (L <= 0) { err = "link_count must be positive"; return false; }
    if (!d.joint_type || !d.joint_parent || !d.joint_q_start || !d.joint_qd_start || !d.joint_X_pj ||
        !d.joint_X_cm || !d.joint_axis || !d.body_I_m) { err = "null joint/body array"; return false; }
    if (d.joint_q_start[L] - d.joint_q_start[0] != Q || d.joint_qd_start[L] - d.joint_qd_start[0] != D) {
        err = "joint_q_start/joint_qd_start sentinels do not match coord/dof counts"; return false;
    }
    static const int kCoords[5] = {1, 1, 4, 0, 7}, kDofs[5] = {1, 1, 3, 0, 6};
    std::vector<int> depth(L, 0);
    int nlev = 0;
    for (int i = 0; i < L; ++i) {
        const int t = d.joint_type[i], p = d.joint_parent[i];
        if (t < 0 || t > 4) { snprintf(buf, sizeof buf, "link %d: unknown joint type %d", i, t); err = buf; return false; }
        if (p >= i || p < -1) { snprintf(buf, sizeof buf, "link %d: parent %d must precede it", i, p); err = buf; return false; }
        if (d.joint_q_start[i + 1] - d.joint_q_start[i] != kCoords[t] || d.joint_qd_start[i + 1] - d.joint_qd_start[i] != kDofs[t]) {
            snprintf(buf, sizeof buf, "link %d: coordinate/dof span does not match joint type %d", i, t); err = buf; return false;
        }
        depth[i] = p < 0 ? 0 : depth[p] + 1;
        if (depth[i] + 1 > nlev) nlev = depth[i] + 1;
        // blockdiag(I_c, m 1) is what the reference builder produces (util.py:340-349)
        const float* I = d.body_I_m + i * 36;
        const float m = I[3 * 6 + 3];
        const float scale = 1e-6f * (1.0f + std::fabs(m));
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) {
                const bool tl = r < 3 && c < 3, br = r >= 3 && c >= 3;
                const float v = I[r * 6 + c];
                if (!tl && !br && std::fabs(v) > scale) { snprintf(buf, sizeof buf, "link %d: body_I_m has off-diagonal blocks", i); err = buf; return false; }
                if (br && std::fabs(v - (r == c ? m : 0.0f)) > scale) { snprintf(buf, sizeof buf, "link %d: body_I_m mass block is not m*1", i); err = buf; return false; }
            }
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < r; ++c)
                if (std::fabs(I[r * 6 + c] - I[c * 6 + r]) > 1e-5f * (std::fabs(I[r * 6 + c]) + std::fabs(I[c * 6 + r]) + 1e-12f)) {
                    snprintf(buf, sizeof buf, "link %d: rotational inertia is not symmetric", i); err = buf; return false;
                }
    }
    for (int k = 0; k < C; ++k) {
        if (d.contact_body0[k] < 0 || d.contact_body0[k] >= L) { err = "contact_body0 out of range (expected env-local link index)"; return false; }
        if (d.contact_material[k] < 0 || d.contact_material[k] >= d.shape_count) { err = "contact_material out of range"; return false; }
    }
    for (int k = 0; k < W; ++k)
        if (d.muscle_links[k] < 0 || d.muscle_links[k] >= L) { err = "muscle_links out of range (expected env-local link index)"; return false; }
    if (M > 0 && (d.muscle_start[0] != 0 || d.muscle_start[M] != W)) { err = "muscle_start must span [0, waypoint_count]"; return false; }

    out = PackHost();
    Pack& h = out.header;
    h = Pack();
    h.L = L; h.D = D; h.Q = Q; h.C = C; h.M = M; h.W = W; h.nlev = nlev;
    h.ground = (d.ground && C > 0) ? 1 : 0;
    h.gx = d.gravity[0]; h.gy = d.gravity[1]; h.gz = d.gravity[2];

    auto push_i = [&](const std::vector<int>& v) { out.int_off.push_back(out.ints.size()); out.ints.insert(out.ints.end(), v.begin(), v.end()); };
    auto push_f = [&](const std::vector<float>& v) {
        while (out.floats.size() % 4) out.floats.push_back(0.0f);
        out.float_off.push_back(out.floats.size()); out.floats.insert(out.floats.end(), v.begin(), v.end());
    };
    const int q0 = d.joint_q_start[0], d0 = d.joint_qd_start[0];
    std::vector<int> type(d.joint_type, d.joint_type + L), parent(d.joint_parent, d.joint_parent + L);
    std::vector<int> qs(L + 1), ds(L + 1);
    for (int i = 0; i <= L; ++i) { qs[i] = d.joint_q_start[i] - q0; ds[i] = d.joint_qd_start[i] - d0; }
    std::vector<int> level_start(nlev + 1, 0), level_links;
    for (int lev = 0; lev < nlev; ++lev) {
        level_start[lev] = (int)level_links.size();
        for (int i = 0; i < L; ++i) if (depth[i] == lev) level_links.push_back(i);
    }
    level_start[nlev] = (int)level_links.size();
    std::vector<int> child_start(L + 1, 0), child_idx;
    for (int i = 0; i < L; ++i) {
        child_start[i] = (int)child_idx.size();
        for (int c = i + 1; c < L; ++c) if (parent[c] == i) child_idx.push_back(c);
    }
    child_start[L] = (int)child_idx.size();
    std::vector<int> anc_start(L + 1, 0), anc_dofs, sub_start(L + 1, 0), sub_links, dof_link(D, 0);
    for (int i = 0; i < L; ++i) {
        anc_start[i] = (int)anc_dofs.size();
        std::vector<int> chain;
        for (int j = i; j >= 0; j = parent[j]) chain.push_back(j);
        for (int k = (int)chain.size() - 1; k >= 0; --k)
            for (int dd = ds[chain[k]]; dd < ds[chain[k] + 1]; ++dd) anc_dofs.push_back(dd);
        for (int dd = ds[i]; dd < ds[i + 1]; ++dd) dof_link[dd] = i;
    }
    anc_start[L] = (int)anc_dofs.size();
    for (int i = 0; i < L; ++i) {
        sub_start[i] = (int)sub_links.size();
        for (int j = i; j < L; ++j) {
            int a = j;
            while (a > i) a = parent[a];
            if (a == i) sub_links.push_back(j);
        }
    }
    sub_start[L] = (int)sub_links.size();
    std::vector<int> path_start(L + 1, 0), path_links;
    for (int i = 0; i < L; ++i) {
        path_start[i] = (int)path_links.size();
        std::vector<int> chain;
        for (int j = i; j >= 0; j = parent[j]) chain.push_back(j);
        for (int k = (int)chain.size() - 1; k >= 0; --k) path_links.push_back(chain[k]);
    }
    path_start[L] = (int)path_links.size();
    // chain decomposition (see dfx_pack.h)
    std::vector<int> nchild(L, 0), chain_of(L, -1), chain_round;
    for (int i = 0; i < L; ++i) if (parent[i] >= 0) ++nchild[parent[i]];
    std::vector<std::vector<int>> chains;
    for (int i = L - 1; i >= 0; --i) {                    // parents precede children: every child's chain exists already
        if (nchild[i] == 1) continue;                     // inner link of a chain: appended when its bottom is visited
        std::vector<int> c;
        int round = 0;
        for (int k = child_start[i]; k < child_start[i + 1]; ++k) {
            const int r = chain_round[chain_of[child_idx[k]]] + 1;
            if (r > round) round = r;
        }
        for (int j = i;;) {
            c.push_back(j);
            chain_of[j] = (int)chains.size();
            const int p = parent[j];
            if (p < 0 || nchild[p] != 1) break;
            j = p;
        }
        chains.push_back(c);
        chain_round.push_back(round);
    }
    int nround = 0;
    for (int r : chain_round) if (r + 1 > nround) nround = r + 1;
    std::vector<int> round_start(nround + 1, 0), chain_start, chain_links;
    for (int r = 0; r < nround; ++r) {
        round_start[r] = (int)chain_start.size();
        for (size_t c = 0; c < chains.size(); ++c) {
            if (chain_round[c] != r) continue;
            chain_start.push_back((int)chain_links.size());
            chain_links.insert(chain_links.end(), chains[c].begin(), chains[c].end());
        }
    }
    round_start[nround] = (int)chain_start.size();
    chain_start.push_back((int)chain_links.size());
    h.nround = nround;
    h.jmask = 0;
    for (int i = 0; i < L; ++i) h.jmask |= 1 << d.joint_type[i];
    h.root_round_single = 1;
    for (size_t c = 0; c < chains.size(); ++c)
        if (chain_round[c] == nround - 1 && (chains[c].size() != 1 || parent[chains[c][0]] >= 0)) h.root_round_single = 0;
    // contacts grouped by body, original order preserved inside a body
    std::vector<int> cbody_start(L + 1, 0), cbody, corder;
    for (int i = 0; i < L; ++i) {
        cbody_start[i] = (int)cbody.size();
        for (int k = 0; k < C; ++k) if (d.contact_body0[k] == i) { cbody.push_back(i); corder.push_back(k); }
    }
    cbody_start[L] = (int)cbody.size();
    std::vector<float> cpoint(C * 3), cdist(C), cmat(C * 4);
    for (int n = 0; n < C; ++n) {
        const int k = corder[n];
        for (int c = 0; c < 3; ++c) cpoint[n * 3 + c] = d.contact_point0[k * 3 + c];
        cdist[n] = d.contact_dist[k];
        for (int c = 0; c < 4; ++c) cmat[n * 4 + c] = d.shape_materials[d.contact_material[k] * 4 + c];
    }
    std::vector<int> mstart(M + 1, 0), mlinks(W);
    for (int i = 0; i <= M && M > 0; ++i) mstart[i] = d.muscle_start[i];
    for (int i = 0; i < W; ++i) mlinks[i] = d.muscle_links[i];
    std::vector<int> aseg_start(M + 1, 0), aseg_way, morder;
    for (int m = 0; m < M; ++m) {
        aseg_start[m] = (int)aseg_way.size();
        for (int i = mstart[m]; i < mstart[m + 1] - 1; ++i) if (mlinks[i] != mlinks[i + 1]) aseg_way.push_back(i);
    }
    if (M > 0) aseg_start[M] = (int)aseg_way.size();
    // muscle groups: same (l0, l1) for every active segment; a group's work (members x active segments) is capped at
    // kMaxEvals segment evaluations and the members of a key are split evenly (SNU: 32 groups of <= 8 evaluations, 96
    // wrench scatters per substep instead of 396)
    constexpr int kMaxEvals = 8;
    std::vector<std::vector<int>> mgroups;
    {
        std::vector<std::vector<int>> keys(M);
        for (int m = 0; m < M; ++m)
            for (int j = aseg_start[m]; j < aseg_start[m + 1]; ++j) { keys[m].push_back(mlinks[aseg_way[j]]); keys[m].push_back(mlinks[aseg_way[j] + 1]); }
        std::vector<char> taken(M, 0);
        for (int m = 0; m < M; ++m) {
            if (taken[m]) continue;
            std::vector<int> same;
            for (int k = m; k < M; ++k) if (!taken[k] && keys[k] == keys[m]) { same.push_back(k); taken[k] = 1; }
            const int nseg = (int)keys[m].size() / 2;
            const int cap = nseg > 0 ? (kMaxEvals / nseg > 0 ? kMaxEvals / nseg : 1) : (int)same.size();
            const int parts = ((int)same.size() + cap - 1) / cap;
            const int base = (int)same.size() / parts, extra = (int)same.size() % parts;
            for (int pi = 0, at = 0; pi < parts; ++pi) {
                const int cnt = base + (pi < extra ? 1 : 0);
                mgroups.emplace_back(same.begin() + at, same.begin() + at + cnt);
                at += cnt;
            }
        }
        // most work first (stable): the first round of item slots gets the long walks, a second one the short ones
        auto work = [&](const std::vector<int>& grp) { return (int)grp.size() * (int)keys[grp[0]].size(); };
        for (size_t a = 1; a < mgroups.size(); ++a)
            for (size_t b = a; b > 0 && work(mgroups[b]) > work(mgroups[b - 1]); --b) std::swap(mgroups[b], mgroups[b - 1]);
    }
    std::vector<int> mgrp_start;
    for (const auto& grp : mgroups) { mgrp_start.push_back((int)morder.size()); morder.insert(morder.end(), grp.begin(), grp.end()); }
    mgrp_start.push_back((int)morder.size());
    h.MG = (int)mgroups.size();
    std::vector<float> Ic(L * 9), mass(L);
    for (int i = 0; i < L; ++i) {
        const float* I = d.body_I_m + i * 36;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Ic[i * 9 + r * 3 + c] = I[r * 6 + c];
        mass[i] = I[3 * 6 + 3];
    }
    push_i(type); push_i(parent); push_i(qs); push_i(ds); push_i(level_start); push_i(level_links);
    push_i(child_start); push_i(child_idx); push_i(anc_start); push_i(anc_dofs); push_i(sub_start);
    push_i(sub_links); push_i(path_start); push_i(path_links); push_i(round_start); push_i(chain_start); push_i(chain_links);
    push_i(dof_link); push_i(cbody_start); push_i(cbody); push_i(mstart); push_i(mlinks); push_i(aseg_start); push_i(aseg_way); push_i(morder); push_i(mgrp_start);
    auto vec = [](const float* p, int n) { return p ? std::vector<float>(p, p + n) : std::vector<float>(n, 0.0f); };
    push_f(vec(d.joint_X_pj, L * 7)); push_f(vec(d.joint_X_cm, L * 7)); push_f(vec(d.joint_axis, L * 3));
    push_f(Ic); push_f(mass);
    push_f(vec(d.joint_target_ke, L)); push_f(vec(d.joint_target_kd, L));
    push_f(vec(d.joint_limit_ke, L)); push_f(vec(d.joint_limit_kd, L));
    push_f(vec(d.joint_target, Q)); push_f(vec(d.joint_limit_lower, Q)); push_f(vec(d.joint_limit_upper, Q));
    push_f(vec(d.joint_armature, D));
    push_f(cpoint); push_f(cdist); push_f(cmat);
    push_f(vec(d.muscle_points, W * 3));
    out.corder = corder;
    out.set_layout_mode(kLayoutLegacy);
    return true;
}

// tape geometry shared by forward / backward / host emulation
struct TapeGeom {
    int N, S, nseg, QD /* floats per (substep, env) row */, DD;
    long long hinv_base;  // float offset of the H^-1 blocks
    long long total;
};
inline TapeGeom tape_geom(int L, int Q, int D, int N, int substeps, int mm_freq, bool bf16 = false) {
    TapeGeom t;
    t.N = N; t.S = substeps; t.QD = dfx_row_units(make_layout(L, D, Q, 0, 0).tape_row, L, D, bf16); t.DD = D * D;
    t.nseg = (substeps + mm_freq - 1) / mm_freq;
    t.hinv_base = (long long)substeps * N * t.QD;
    t.total = t.hinv_base + (long long)t.nseg * N * t.DD;
    return t;
}

}  // namespace dfx
