"""Seeded random articulations as model dicts (the field names of tests/golden/*.npz model/*, one environment), so that
articulation_from_model, Oracle.from_model, EmuSim and ArticulationEngine take them unchanged, plus batches of states
for them in the format of exact_util.make_batch.

Two families:
* size twins: exactly the (L, D, Q, C, M) and joint-type mask of a DiffRL articulation, so that they run on that
  articulation's tile kernel and lane-group specialisation -- with a different tree, different frames, inertias, gains,
  limits and contact placement;
* generic models: no specialisation exists for them -- all five joint types mixed, free / fixed / planar roots, L from 2
  to 40, D above 32 (a lane group loops over more items than it has lanes), a forest of two roots.

Tree orders are random topological orders (parents precede children, as dfx_pack_create requires), not depth-first."""
import os
import sys
from concurrent.futures import ProcessPoolExecutor
import multiprocessing

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE, os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import exact_util as X  # noqa: E402
from oracle import Oracle  # noqa: E402

PRISMATIC, REVOLUTE, BALL, FIXED, FREE = 0, 1, 2, 3, 4
NQ, ND = (1, 1, 4, 0, 7), (1, 1, 3, 0, 6)
DT_SUB = 1.0 / 960.0          # the substep of every DiffRL locomotion env (dt 1/60, 16 substeps)


# ------------------------------------------------------------------ quaternions / transforms (x, y, z, w), float64
def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _qrot(q, v):
    return X._quat_rotate(q, v)


def _axis_angle(axis, ang):
    axis = np.asarray(axis, np.float64)
    return np.concatenate([axis * np.sin(ang / 2), [np.cos(ang / 2)]])


def _unit(rng):
    v = rng.standard_normal(3)
    return v / np.linalg.norm(v)


def _rot(rng, max_angle):
    return _axis_angle(_unit(rng), rng.uniform(0.0, max_angle))


# ------------------------------------------------------------------ trees
def _topological(rng, parent_of):
    """relabel a tree (parent_of[i] for a tree in any labelling, -1 for roots) in a random topological order: parents
    precede children, siblings and subtrees interleave (not depth-first).  Returns (new parent array, old -> new)."""
    L = len(parent_of)
    children = [[] for _ in range(L)]
    for i, p in enumerate(parent_of):
        if p >= 0:
            children[p].append(i)
    ready = [i for i in range(L) if parent_of[i] < 0]
    order = []
    while ready:
        k = ready.pop(int(rng.integers(len(ready))) if len(order) else 0)   # the first root stays link 0
        order.append(k)
        ready += children[k]
    new = {old: n for n, old in enumerate(order)}
    return [(-1 if parent_of[old] < 0 else new[parent_of[old]]) for old in order], new


def _random_tree(rng, L, roots=1, one_child_root=False, wide_at=None, deep=False):
    """parent array (in creation order) of a random forest of L links.  one_child_root: the root has one child above the
    first branch; wide_at: a link at depth >= 2 with 3+ children; deep: mostly a chain."""
    parent = [-1] * roots
    depth = [0] * roots
    while len(parent) < L:
        n = len(parent)
        if one_child_root and n == roots:
            p = 0
        elif deep and rng.uniform() < 0.8:
            p = n - 1
        else:
            cand = [i for i in range(n) if not (one_child_root and i == 0)] or [0]
            p = int(rng.choice(cand))
        parent.append(p)
        depth.append(depth[p] + 1)
    if wide_at is not None and L >= 8:
        # three (more) children for the first link at depth >= 2 that has a later sibling-free slot: re-hang leaves
        hubs = [i for i in range(L) if depth[i] >= 2]
        if hubs:
            hub = hubs[0]
            leaves = [i for i in range(L) if i > hub and i not in parent and parent[i] != hub]
            for leaf in leaves[:3]:
                parent[leaf] = hub
    return parent


# ------------------------------------------------------------------ model dicts
class RandomModel:
    """model: the model dict; name; (S, mm, dt): the env-step pattern the model is stepped with by default;
    height: [(coordinate, links of its subtree)] the coordinates that move a root vertically (free / planar roots);
    twin_of: the DiffRL articulation whose sizes it copies, or None."""

    def __init__(self, name, model, S, mm, twin_of, height):
        self.name, self.model, self.S, self.mm, self.twin_of, self.height = name, model, S, mm, twin_of, height
        self.dt = DT_SUB * S

    def patterns(self):
        """(substeps, mass-matrix period): the default, one substep, and (7, 3) (a short last segment)"""
        return list(dict.fromkeys([(self.S, self.mm), (1, 1), (7, 3)]))

    def pattern_dt(self, S):
        return DT_SUB * S


def _build(rng, types, parent, contacts, muscles=0, root_frames=None):
    """types / parent: per link (parents precede children); contacts: list of body indices; root_frames: {link: X_pj}."""
    L = len(types)
    qs, ds = [0], [0]
    for t in types:
        qs.append(qs[-1] + NQ[t]); ds.append(ds[-1] + ND[t])
    Q, D = qs[-1], ds[-1]
    X_pj = np.zeros((L, 7)); X_cm = np.zeros((L, 7)); axis = np.zeros((L, 3)); I_m = np.zeros((L, 6, 6))
    tke, tkd, lke, lkd = (np.zeros(L) for _ in range(4))
    target, lower, upper = np.zeros(Q), np.full(Q, -1e6), np.full(Q, 1e6)
    arm = np.zeros(D)
    for i, t in enumerate(types):
        if parent[i] < 0:
            X_pj[i] = (root_frames or {}).get(i, np.array([0, 0, 0, 0, 0, 0, 1.0]))
        else:
            X_pj[i, :3] = _unit(rng) * rng.uniform(0.08, 0.3)
            X_pj[i, 3:] = _rot(rng, np.pi) if rng.uniform() < 0.5 else _rot(rng, 0.4)
        X_cm[i, :3] = _unit(rng) * rng.uniform(0.0, 0.08)
        X_cm[i, 3:] = _rot(rng, 0.5)
        axis[i] = _unit(rng)
        m = rng.uniform(1.0, 8.0)
        R = np.array([_qrot(_rot(rng, np.pi), e) for e in np.eye(3)]).T
        Ic = R @ np.diag(m * rng.uniform(0.003, 0.03, 3)) @ R.T
        I_m[i, :3, :3] = (Ic + Ic.T) / 2
        I_m[i, 3:, 3:] = m * np.eye(3)
        if t in (PRISMATIC, REVOLUTE):
            c, d = qs[i], ds[i]
            lke[i], lkd[i] = rng.uniform(200, 1000), rng.uniform(0.5, 5)
            tke[i], tkd[i] = rng.uniform(0, 20), rng.uniform(0.1, 3)
            span = (0.05, 0.3) if t == PRISMATIC else (0.2, 1.4)
            lower[c], upper[c] = -rng.uniform(*span), rng.uniform(*span)
            target[c] = rng.uniform(lower[c], upper[c]) / 2
            arm[d] = rng.uniform(0.02, 0.2)
        elif t == BALL:
            tke[i], tkd[i] = rng.uniform(0, 10), rng.uniform(0.1, 3)
            arm[ds[i]:ds[i + 1]] = rng.uniform(0.02, 0.2, 3)
    C = len(contacts)
    n_mat = int(rng.integers(1, 4))
    mats = np.stack([rng.uniform(2e3, 2e4, n_mat), rng.uniform(100, 1000, n_mat), rng.uniform(50, 500, n_mat),
                     rng.uniform(0.25, 1.0, n_mat)], axis=1)
    body0 = np.asarray(contacts, np.int32)
    point0 = np.array([_unit(rng) * rng.uniform(0.0, 0.25) for _ in range(C)]).reshape(C, 3)
    cdist = rng.uniform(0.0, 0.06, C)
    cmat = rng.integers(0, n_mat, C).astype(np.int32)
    # muscles: 2-4 way-points, from an ancestor down a tree path (up to three links long) to a descendant
    mstart, mlinks, mpoints = [0], [], []
    for _ in range(muscles):
        path = [int(rng.integers(1, L)) if L > 1 else 0]
        while parent[path[-1]] >= 0 and len(path) < 4:
            path.append(parent[path[-1]])
        for k in sorted(rng.integers(0, len(path), int(rng.integers(2, 5))))[::-1]:
            mlinks.append(path[k]); mpoints.append(_unit(rng) * rng.uniform(0.02, 0.2))
        mstart.append(len(mlinks))
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(
        joint_type=np.asarray(types, np.int32), joint_parent=np.asarray(parent, np.int32),
        joint_q_start=np.asarray(qs, np.int32), joint_qd_start=np.asarray(ds, np.int32),
        joint_X_pj=f32(X_pj), joint_X_cm=f32(X_cm), joint_axis=f32(axis), body_I_m=f32(I_m),
        joint_target_ke=f32(tke), joint_target_kd=f32(tkd), joint_limit_ke=f32(lke), joint_limit_kd=f32(lkd),
        joint_target=f32(target), joint_limit_lower=f32(lower), joint_limit_upper=f32(upper), joint_armature=f32(arm),
        contact_body0=body0, contact_point0=f32(point0), contact_dist=f32(cdist), contact_material=cmat,
        shape_materials=f32(mats), muscle_start=np.asarray(mstart, np.int32), muscle_links=np.asarray(mlinks, np.int32),
        muscle_points=f32(np.array(mpoints).reshape(-1, 3)), gravity=np.array([0.0, -9.81, 0.0], np.float32),
        articulation_joint_start=np.array([0, L], np.int32), ground=True)


def _contacts(rng, L, C, mode):
    """contact bodies: spread over the links ('spread'), including the root ('root'), or all on one link ('one')"""
    if mode == "one":
        return [int(rng.integers(0, L))] * C
    out = rng.integers(0, L, C).tolist()
    if mode == "root":
        out[: max(1, C // 4)] = [0] * max(1, C // 4)
    return out


def _assemble(rng, root_types, body_types, tree_parent, contacts, muscles=0, planar=False):
    """root_types: the root chain (a free link, a planar P-P-R chain or a fixed link) at links 0..; body_types: the other
    links, hung below by tree_parent (indices into the body links, -1 = the last root-chain link)."""
    nr = len(root_types)
    parent_of = list(range(-1, nr - 1)) + [(nr - 1 if p < 0 else nr + p) for p in tree_parent]
    types0 = list(root_types) + list(body_types)
    parent, new = _topological(rng, parent_of)
    types = [None] * len(types0)
    for old, n in new.items():
        types[n] = types0[old]
    return types, parent


# ------------------------------------------------------------------ the two families
TWINS = ["AntEnv", "HumanoidEnv", "HopperEnv", "CheetahEnv", "CartPoleSwingUpEnv", "SNUHumanoidEnv"]
GENERIC = ["pair", "mixed", "planar", "fixed", "forest", "deep24", "wide40"]


def twin(name, seed=0):
    rng = np.random.default_rng([seed, TWINS.index(name)])
    S, mm, _ = X.config(name)
    planar_axes = None
    if name in ("AntEnv", "HumanoidEnv"):
        L, C = (9, 25) if name == "AntEnv" else (22, 35)
        tree = _random_tree(rng, L, one_child_root=(name == "HumanoidEnv"), wide_at=True)
        parent, _ = _topological(rng, tree)
        types = [FREE] + [REVOLUTE] * (L - 1)
        contacts = _contacts(rng, L, C, "root" if name == "AntEnv" else "spread")
    elif name == "SNUHumanoidEnv":
        tree = _random_tree(rng, 11, wide_at=True)
        parent, _ = _topological(rng, tree)
        rest = [BALL] * 4 + [REVOLUTE] * 6
        rng.shuffle(rest)
        types = [FREE] + rest
        contacts = _contacts(rng, 11, 88, "spread")
    elif name in ("HopperEnv", "CheetahEnv"):
        L, C = (6, 8) if name == "HopperEnv" else (9, 16)
        body = [REVOLUTE] * (L - 3)
        body[int(rng.integers(1, L - 3))] = PRISMATIC          # a slider below a rotation
        tree = [-1] + [int(rng.integers(-1, k)) for k in range(1, L - 3)]
        types, parent = _assemble(rng, [PRISMATIC, PRISMATIC, REVOLUTE], body, tree, None)
        planar_axes = True
        contacts = _contacts(rng, L, C, "one" if name == "HopperEnv" else "spread")
        contacts = [c if c >= 2 else int(rng.integers(2, L)) for c in contacts]     # (the root sliders carry no shapes)
    else:   # CartPole: a fixed link, a slider and a hinge, the fixed link in the middle of the tree
        types, parent, contacts = [PRISMATIC, FIXED, REVOLUTE], [-1, 0, 1], []
    model = _build(rng, types, parent, contacts, muscles=152 if name == "SNUHumanoidEnv" else 0)
    if planar_axes:
        _make_planar(model)
    if name == "CartPoleSwingUpEnv":
        model["joint_X_pj"][0] = [0, 2.0, 0, 0, 0, 0, 1]
    return RandomModel("twin_" + name, model, S, mm, name, _heights(model))


def _make_planar(model):
    """links 0, 1, 2 become the planar root: slider along world x, slider along world y, hinge about world z"""
    model["joint_axis"][0:3] = [[1, 0, 0], [0, 1, 0], [0, 0, 1]]
    model["joint_X_pj"][0:3] = [0, 0, 0, 0, 0, 0, 1]
    model["joint_X_cm"][0:2] = [0, 0, 0, 0, 0, 0, 1]
    model["body_I_m"][0:2] *= 0.2                      # light carriage links (the DiffRL ones are massless with armature)
    for i in range(3):
        c = model["joint_q_start"][i]
        model["joint_limit_lower"][c], model["joint_limit_upper"][c], model["joint_target"][c] = -1e6, 1e6, 0.0
        model["joint_target_ke"][i] = model["joint_target_kd"][i] = 0.0
        model["joint_armature"][model["joint_qd_start"][i]] = 0.1


def generic(kind, seed=0):
    rng = np.random.default_rng([seed, 100 + GENERIC.index(kind)])
    if kind == "pair":          # L = 2: a free root and a ball joint, contacts on both
        types, parent, contacts = [FREE, BALL], [-1, 0], _contacts(rng, 2, 6, "root")
    elif kind == "mixed":       # every joint type; a fixed link in the middle of the tree with children and contacts
        body = [REVOLUTE, BALL, PRISMATIC, FIXED, REVOLUTE, BALL, REVOLUTE, PRISMATIC, REVOLUTE, REVOLUTE, BALL]
        tree = [-1, 0, 1, 0, 3, 3, 3, 4, 5, 1, 9]                # ball below a hinge, slider below a rotation, the
        types, parent = _assemble(rng, [FREE], body, tree, None)   # fixed link (body 3) with three children
        fixed = types.index(FIXED)
        contacts = _contacts(rng, len(types), 14, "spread") + [fixed] * 3
    elif kind == "planar":      # planar root, depth-2 branch point with three children, mixed joints below
        body = [REVOLUTE, REVOLUTE, BALL, PRISMATIC, REVOLUTE, REVOLUTE, REVOLUTE]
        tree = [-1, 0, 1, 1, 1, 2, 4]
        types, parent = _assemble(rng, [PRISMATIC, PRISMATIC, REVOLUTE], body, tree, None)
        contacts = [c if c >= 3 else int(rng.integers(3, len(types))) for c in _contacts(rng, len(types), 12, "spread")]
    elif kind == "fixed":       # a fixed root hanging a deep chain with a side branch; no ground contact, limits only
        body = [REVOLUTE, PRISMATIC, BALL, REVOLUTE, REVOLUTE, REVOLUTE, PRISMATIC, REVOLUTE, REVOLUTE, BALL, REVOLUTE,
                REVOLUTE, REVOLUTE]
        tree = [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 3]          # chain of 12 (deeper than Humanoid's 9) + a branch
        types, parent = _assemble(rng, [FIXED], body, tree, None)
        contacts = []
    elif kind == "forest":      # two roots in one environment: a free body with legs and a planar hopper
        tree1 = [-1, 0, 0, 0, 1, 2]
        types1 = [FREE, REVOLUTE, REVOLUTE, BALL, REVOLUTE, REVOLUTE, REVOLUTE]
        par1 = [-1] + [0 if p < 0 else p + 1 for p in tree1]
        types2 = [PRISMATIC, PRISMATIC, REVOLUTE, REVOLUTE, PRISMATIC]
        par2 = [-1, 0, 1, 2, 3]
        types0 = types1 + types2
        parent_of = par1 + [(-1 if p < 0 else p + len(types1)) for p in par2]
        parent, new = _topological(rng, parent_of)
        types = [None] * len(types0)
        for old, n in new.items():
            types[n] = types0[old]
        second = new[len(types1)]
        contacts = [new[k] for k in rng.integers(0, len(types1), 8)] + [new[len(types1) + 3], new[len(types1) + 4]] * 3
        model = _build(rng, types, parent, contacts)
        model["joint_X_pj"][second] = [1.5, 0, 0, 0, 0, 0, 1]         # side by side
        k = new[len(types1) + 1]
        model["joint_axis"][second], model["joint_axis"][k] = [1, 0, 0], [0, 1, 0]
        model["joint_X_pj"][k] = [0, 0, 0, 0, 0, 0, 1]
        model["joint_X_pj"][new[len(types1) + 2]] = [0, 0, 0, 0, 0, 0, 1]
        model["joint_axis"][new[len(types1) + 2]] = [0, 0, 1]
        for i in (second, k):
            c = model["joint_q_start"][i]
            model["joint_limit_lower"][c], model["joint_limit_upper"][c], model["joint_target"][c] = -1e6, 1e6, 0.0
            model["joint_target_ke"][i] = 0.0
        return RandomModel("gen_" + kind, model, 8, 4, None, _heights(model))
    elif kind == "deep24":      # 24 links, 8 balls: D = 6 + 24 + 15 = 45 > 32
        body = [BALL] * 8 + [REVOLUTE] * 13 + [PRISMATIC] * 2
        rng.shuffle(body)
        tree = [int(p) - 1 for p in _random_tree(rng, len(body) + 1, deep=True)[1:]]
        types, parent = _assemble(rng, [FREE], body, tree, None)
        contacts = _contacts(rng, len(types), 30, "spread")
    else:                       # wide40: 40 links (30 hinges, 6 balls, 3 fixed), D = 6 + 30 + 6 * 3 = 54
        body = [BALL] * 6 + [REVOLUTE] * 30 + [FIXED] * 3
        rng.shuffle(body)
        tree = [int(p) - 1 for p in _random_tree(rng, len(body) + 1, one_child_root=True, wide_at=True)[1:]]
        types, parent = _assemble(rng, [FREE], body, tree, None)
        contacts = _contacts(rng, len(types), 40, "spread")
    model = _build(rng, types, parent, contacts)
    if kind == "planar":
        _make_planar(model)
    if kind == "fixed":
        model["joint_X_pj"][0] = [0, 3.0, 0, 0, 0, 0, 1]
    return RandomModel("gen_" + kind, model, 8, 4, None, _heights(model))


def all_models(seed=0):
    return [twin(n, seed) for n in TWINS] + [generic(k, seed) for k in GENERIC]


# ------------------------------------------------------------------ kinematics (float64) and states
def _subtree(parent, r):
    out = []
    for j in range(len(parent)):
        a = j
        while a > r:
            a = parent[a]
        if a == r:
            out.append(j)
    return out


def _heights(model):
    """[(height coordinate, links it lifts)]: a free root's y, a planar root's world-y slider (links 0, 1, 2 of a
    P-P-R chain with axes x, y, z)"""
    t, par, qs = model["joint_type"], model["joint_parent"], model["joint_q_start"]
    out = []
    for r in np.nonzero(par < 0)[0]:
        if t[r] == FREE:
            out.append((int(qs[r]) + 1, _subtree(par, r)))
        elif t[r] == PRISMATIC:
            k = [j for j in range(len(t)) if par[j] == r][0]
            if t[k] == PRISMATIC and abs(model["joint_axis"][k][1]) > 0.99:
                out.append((int(qs[k]), _subtree(par, r)))
    return out


def body_transforms(model, q):
    """X_sc of every link (float64 [L, 7]) at coordinates q"""
    t, par, qs = model["joint_type"], model["joint_parent"], model["joint_q_start"]
    out = np.zeros((len(t), 7))
    for i in range(len(t)):
        Xpj = np.asarray(model["joint_X_pj"][i], np.float64)
        ax, c = np.asarray(model["joint_axis"][i], np.float64), int(qs[i])
        jp, jq = np.zeros(3), np.array([0, 0, 0, 1.0])
        if t[i] == PRISMATIC:
            jp = ax * q[c]
        elif t[i] == REVOLUTE:
            jq = _axis_angle(ax, q[c])
        elif t[i] == BALL:
            jq = np.asarray(q[c:c + 4], np.float64)
        elif t[i] == FREE:
            jp, jq = np.asarray(q[c:c + 3], np.float64), np.asarray(q[c + 3:c + 7], np.float64)
        p, r = Xpj[:3] + _qrot(Xpj[3:], jp), _qmul(Xpj[3:], jq)
        if par[i] >= 0:
            P = out[par[i]]
            p, r = P[:3] + _qrot(P[3:], p), _qmul(P[3:], r)
        out[i, :3], out[i, 3:] = p, r
    return out


def contact_heights(model, q):
    Xs = body_transforms(model, q)
    return np.array([(Xs[b, :3] + _qrot(Xs[b, 3:], model["contact_point0"][k]))[1] - model["contact_dist"][k]
                     for k, b in enumerate(model["contact_body0"])])


def random_state(rm, rng, clearance, vscale=0.5):
    """one environment: joints uniformly within 0.8x their limits, balls and free roots turned by up to ~0.5 rad, random
    velocities of scale vscale; each free / planar root lifted so that its subtree's lowest contact point sits `clearance` above the ground"""
    m = rm.model
    t, qs, ds = m["joint_type"], m["joint_q_start"], m["joint_qd_start"]
    Q, D = int(qs[-1]), int(ds[-1])
    q, qd = np.zeros(Q), vscale * rng.standard_normal(D)
    for i in range(len(t)):
        c = int(qs[i])
        if t[i] in (PRISMATIC, REVOLUTE):
            lo, hi = float(m["joint_limit_lower"][c]), float(m["joint_limit_upper"][c])
            q[c] = rng.uniform(0.8 * lo, 0.8 * hi) if hi < 1e5 else rng.uniform(-0.3, 0.3)
        elif t[i] == BALL:
            q[c:c + 4] = _rot(rng, 0.5)
        elif t[i] == FREE:
            q[c:c + 3] = [rng.uniform(-0.5, 0.5), 0.0, rng.uniform(-0.5, 0.5)]
            q[c + 3:c + 7] = _rot(rng, 0.5)
    if len(m["contact_body0"]):
        h = contact_heights(m, q)
        for coord, links in rm.height:
            mine = [k for k, b in enumerate(m["contact_body0"]) if b in links]
            if mine:
                q[coord] += clearance - h[mine].min()
    return q.astype(np.float32), qd.astype(np.float32)


def make_batch(rm, n_total, n_exact, seed=0):
    """n_total environments of random states (contacts from 2 cm inside the ground to 6 cm above it, a quarter of them
    nearly at rest: friction below its Coulomb cap) with
    exact_util.regime_rows (pushes into every limit, into the ground with sliding, into the air, actions at +-1.5x their
    range) at n_exact spread positions; the format of exact_util.make_batch: (desc, inputs, sample indices)."""
    o = oracle(rm)
    desc = o.desc
    Q, D, M = desc.Q, desc.D, desc.M
    rng = np.random.default_rng([seed, 7])
    act_range = rng.uniform(0.5, 3.0, D).astype(np.float32)
    musc_range = np.ones(M, np.float32) if M else None
    states = [random_state(rm, rng, rng.uniform(-0.02, 0.06), 0.02 if k % 4 == 0 else 0.5) for k in range(n_total)]
    q = np.stack([s[0] for s in states]); qd = np.stack([s[1] for s in states])
    a = (act_range * rng.uniform(-1, 1, (n_total, D))).astype(np.float32)
    m = rng.uniform(0, 1, (n_total, M)).astype(np.float32) if M else None
    sample = np.unique(np.linspace(0, n_total - 1, n_exact).round().astype(np.int64))
    bq, bqd = random_state(rm, rng, 0.005)
    regime = X.regime_rows(desc, bq, bqd, a[0].copy(), None if M == 0 else m[0].copy(), act_range, musc_range)
    assert len(regime) <= len(sample), (rm.name, len(regime), len(sample))
    slots = sample[np.linspace(0, len(sample) - 1, len(regime)).round().astype(np.int64)] if regime else []
    for i, (rq, rqd, ra, rmu) in zip(slots, regime):
        q[i], qd[i], a[i] = rq, rqd, ra
        if M:
            m[i] = rmu
    inp = dict(q0=q, qd0=qd, act=a, musc=m, gq_out=rng.standard_normal((n_total, Q)).astype(np.float32),
               gqd_out=rng.standard_normal((n_total, D)).astype(np.float32))
    return desc, inp, sample


# ------------------------------------------------------------------ oracle and exact gradients (process pool)
_oracles = {}


def _spec_model(spec):
    fam, name, seed = spec
    return twin(name, seed) if fam == "twin" else generic(name, seed)


def spec(rm, seed=0):
    return ("twin", rm.twin_of, seed) if rm.twin_of else ("generic", rm.name[len("gen_"):], seed)


def oracle(rm):
    if rm.name not in _oracles:
        _oracles[rm.name] = Oracle.from_model(rm.model, 1)
    return _oracles[rm.name]


_spec_oracles = {}


def _exact_job(job):
    sp, S, mm, dt, q, qd, a, m, gq, gqd = job
    if sp not in _spec_oracles:
        _spec_oracles[sp] = Oracle.from_model(_spec_model(sp).model, 1)
    return _spec_oracles[sp].exact_gradient(q, qd, a, m, gq, gqd, S, mm, dt)


_cache = {}


def exact_gradients(rm, inp, idx, S, mm, dt, seed=0):
    """[gq, gqd, gact(, gmusc)] as [len(idx), w] fp64 arrays: the complex-step gradients of environments idx"""
    key = (rm.name, seed, S, mm, dt, tuple(int(i) for i in idx)) + tuple(inp[k][idx].tobytes() for k in ("q0", "qd0", "act", "gq_out", "gqd_out"))
    if key in _cache:
        return _cache[key]
    m = inp["musc"]
    sp = spec(rm, seed)
    jobs = [(sp, S, mm, dt, inp["q0"][i], inp["qd0"][i], inp["act"][i], None if m is None else m[i], inp["gq_out"][i],
             inp["gqd_out"][i]) for i in idx]
    workers = max(1, min(16, len(os.sched_getaffinity(0)), len(jobs)))
    if workers == 1:
        res = [_exact_job(j) for j in jobs]
    else:
        with ProcessPoolExecutor(workers, mp_context=multiprocessing.get_context("spawn")) as pool:
            res = list(pool.map(_exact_job, jobs, chunksize=max(1, len(jobs) // (4 * workers))))
    out = [np.stack([r[k] for r in res]) for k in range(4 if res[0][3] is not None else 3)]
    _cache[key] = out
    return out


# ------------------------------------------------------------------ a random tree through the public dflex API
def builder_model(adapter, seed=0):
    """A random articulation built with dflex.sim.ModelBuilder (add_articulation / add_link / add_shape_capsule /
    add_shape_box, finalize, collide): a free root and 9 links of every other joint type hung below random earlier links
    (parents precede children, not depth-first), each carrying a capsule or a box in a random pose.  Returns (Model, one
    state (q, qd, act) as float32 arrays with the root lowered until its lowest contact point is 1 cm inside the ground)."""
    import dflex as df
    from diffrl_b200.modelpack import articulation_from_model
    rng = np.random.default_rng([seed, 200])
    u = df.util
    b = df.sim.ModelBuilder()
    b.add_articulation()
    root = b.add_link(-1, u.transform((0.0, 1.0, 0.0), u.quat_identity()), (0.0, 0.0, 0.0), df.sim.JOINT_FREE, armature=0.0)
    b.add_shape_box(root, hx=0.2, hy=0.08, hz=0.15, density=300.0, ke=1e4, kd=300.0, kf=200.0, mu=0.8)
    links = [root]
    for t in (REVOLUTE, BALL, PRISMATIC, FIXED, REVOLUTE, REVOLUTE, BALL, PRISMATIC, REVOLUTE):
        parent = int(rng.choice(links))
        X = u.transform(tuple(_unit(rng) * rng.uniform(0.1, 0.3)), tuple(_rot(rng, np.pi)))
        span = 0.2 if t == PRISMATIC else 1.0
        link = b.add_link(parent, X, tuple(_unit(rng)), t, armature=float(rng.uniform(0.02, 0.1)), stiffness=float(rng.uniform(0, 10)),
                          damping=float(rng.uniform(0.1, 2)), limit_lower=-span * float(rng.uniform(0.3, 1)),
                          limit_upper=span * float(rng.uniform(0.3, 1)), limit_ke=float(rng.uniform(200, 1000)),
                          limit_kd=float(rng.uniform(1, 5)))
        pos, rot = tuple(_unit(rng) * rng.uniform(0.0, 0.1)), tuple(_rot(rng, np.pi))
        if len(links) % 2:
            b.add_shape_capsule(link, pos=pos, rot=rot, radius=0.04, half_width=0.1, density=500.0, ke=1e4, kd=300.0, kf=200.0, mu=0.8)
        else:
            b.add_shape_box(link, pos=pos, rot=rot, hx=0.05, hy=0.04, hz=0.06, density=500.0, ke=1e4, kd=300.0, kf=200.0, mu=0.8)
        links.append(link)
    model = b.finalize(adapter)
    model.ground = True
    model.collide(model.state())
    desc, _ = articulation_from_model(model, 1)
    a = desc.arrays
    q = model.joint_q.detach().cpu().numpy().astype(np.float64)
    for i, t in enumerate(a["joint_type"]):
        c = int(a["joint_q_start"][i])
        if t in (PRISMATIC, REVOLUTE):
            q[c] = rng.uniform(0.8 * a["joint_limit_lower"][c], 0.8 * a["joint_limit_upper"][c])
        elif t == BALL:
            q[c:c + 4] = _rot(rng, 0.5)
    q[3:7] = _rot(rng, 0.4)
    heights = contact_heights(a, q)
    q[1] += -0.01 - heights.min()
    qd = 0.5 * rng.standard_normal(desc.D)
    act = rng.uniform(-2, 2, desc.D)
    return model, (q.astype(np.float32), qd.astype(np.float32), act.astype(np.float32))
