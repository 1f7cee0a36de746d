"""TEST-ONLY probe envs that read the physics state a custom reward sees, and its fp64 reference.

The probe reward (tests/probes/state_probe_reward.cuh) returns, at env step s, element
e(s) = (user[0] + s user[1]) mod E of the flat order ``LAYOUT`` of the reward contract
(include/dial_custom_reward.h), as the kernel holds it:
  qpos[nq], qvel[nv],
  per body b = 0 .. nbody-1 (the world included): xpos[3], xquat[4], xmat[9], dial_xd_ang[3], dial_xd_vel[3],
  per contact: contact_dist, contact_pos[3],
  per site: dial_site_xpos[3].
A rollout of explicit actions then reads one element per row and step, and the reference is recomputed
in fp64 by oracle/mjx_oracle.py from the kernel's own stored states: the kinematic fields of step t from
the state the step started from (q[t-1], qd[t-1], or the start state at t = 0), as the contract promises;
qpos / qvel from the state after it (q[t], qd[t]), bit for bit.  Kinematic fields are compared with one
physics substep per env step: the pre-state of the last of several substeps is never stored.

Tolerance of one element (``reference``), first-order fp32 error propagation with e = 2^-24, evaluated on
the fp64 reference state and used as it is:
  rotation   th_b = th_parent + 8 e (one quaternion product, rotation and normalisation per level)
             + ulp(dq) + 4 s(dq / 2) per hinge: the kernel forms dq = qpos - qpos0 in fp32 (half an ulp),
             and its sin / cos of dq / 2 have absolute error s; a free joint's normalised quaternion
             starts at 8 e.  s = 2 e for libm (the CPU warp emulator); on the GPU the SFU's __sincosf,
             2^-21.41 for |x| <= pi plus 2 ulp(x) for its fp32 range reduction, which grows with the angle.
  xquat      2 th_b + 2 e;  xmat 4 th_b + 4 e (products of two quaternion components).
  xpos       dx_b = dx_parent + L_b th_b + 4 e (|xpos_b| + L_b), L_b = |body_pos| + 2 |jnt_pos| (+ |dq| of a
             slide joint): the chain's offsets rotated by the accumulated rotation error; 0 for a free root.
  a point p on body b at offset o (xipos, a geom centre, dial_site_xpos): dx_b + 4 th_b |o| + 4 e (|p| + |o|).
  subtree COM of a tree: the largest xipos bound of its bodies + 2 e n_tree max |xipos|.
  dial_xd_ang  sum over the dofs j of the chain of |qd_j| (2 th_j + 4 e) + 2 e n_chain |ang|.
  dial_xd_vel  the helper transports cvel_lin = sum_j qd_j axis_j x (com - anchor_j) from the subtree COM
             to the body origin x; the kernel's fp32 COM is one value in both terms and cancels, so the result
             is sum_j qd_j axis_j x (x - anchor_j) up to rounding: sum over the rotational dofs j of
             |qd_j| (2 th_j |x - anchor_j| + dx + d(anchor_j) + 4 e (|com| + |anchor_j|))
             + (2 n_chain + 4) e (|cvel_lin| + |x - com| |ang|), the last term the rounding of the cancellation.
  contacts   plane-sphere / plane-capsule: the sphere or capsule-end centre c (the capsule axis adds
             hl (4 th + 4 e)), dist dc + 4 th_plane |c - plane| + d(plane) + 4 e (|c| + |plane| + r),
             pos dc + d(dist) / 2 + 4 th_plane r + 4 e (|pos| + r).
             sphere-sphere / sphere-capsule / capsule-capsule: the closest points q1, q2 (clipped
             projections: 1-Lipschitz), dist d(q1) + d(q2) + 4 e (|q2 - q1| + r1 + r2), the normal
             n = (q2 - q1) / |q2 - q1| to 2 (d(q1) + d(q2) + 4 e |q2 - q1|) / |q2 - q1| (at most 2; exact
             at coincident centres, where both take the fallback normal), pos d(q1) + |r1 + dist / 2| d(n)
             + d(dist) / 2 + 4 e |pos|.  Capsule-capsule closest points are ill-conditioned as the axes
             become parallel: the segment parameters move by (2 d(base) + 4 (|trans| + ha + hb) d(axis)) /
             (1 - (a.b)^2 + 1e-6), at most 2 (ha + hb) (the two candidate pairs may swap), added to q1, q2
             for contact_pos only; the distance between the segments stays well conditioned.  Allegro's
             fingertip capsules are near parallel in ordinary poses (1 - (a.b)^2 ~ 1e-4 at its initial pose),
             so there contact_pos often sits at the cap and is checked only to the capsules' length;
             contact_dist stays tight.
The bounds are first order: the products of two error terms they drop are below e^2 relative.  The worst
ratios measured are listed in tests/test_gpu_state_probe.py."""
import copy
import functools
import os
import sys
import tempfile

import numpy as np

from tests.conftest import ROOT

PROBE = os.path.join(ROOT, "tests", "probes", "state_probe_reward.cuh")
EX = os.path.join(ROOT, "dial_mpc_b200", "examples", "custom_env")
MODELS = os.path.join(ROOT, "tests", "models")
E32 = 2.0 ** -24
BODY_FIELDS = (("xpos", 3), ("xquat", 4), ("xmat", 9), ("xd_ang", 3), ("xd_vel", 3))
NB = sum(n for _, n in BODY_FIELDS)     # 22 floats per body


def _pair_names():
    """{kind: name} of the oracle's PAIR_* constants (oracle/mjx_oracle.py)."""
    from oracle import mjx_oracle as mo
    return {v: k[5:].lower().replace("_", "-") for k, v in vars(mo).items() if k.startswith("PAIR_")}


PAIR_NAMES = _pair_names()


def kernel_pair_kinds():
    """{name: kind} of the PAIR_* enum of the device code (dial_device.cuh)."""
    import re
    src = open(os.path.join(ROOT, "dial_mpc_b200", "csrc", "dial_device.cuh")).read()
    enum = re.search(r"enum\s*\{([^}]*PAIR_[^}]*)\}", src).group(1)
    return {k[5:].lower().replace("_", "-"): int(v) for k, v in re.findall(r"(PAIR_\w+)\s*=\s*(\d+)", enum)}


# ---- the flat element order ---------------------------------------------------------------------------
def n_elements(m):
    return m.nq + m.nv + NB * m.nbody + 4 * m.ncon + 3 * m.nsite


def layout(m):
    """[(field, index...)] of every element, in the probe's order."""
    out = [("qpos", i) for i in range(m.nq)] + [("qvel", i) for i in range(m.nv)]
    for b in range(m.nbody):
        for f, n in BODY_FIELDS:
            out += [(f, b, k) for k in range(n)]
    for c in range(m.ncon):
        out += [("contact_dist", c)] + [("contact_pos", c, k) for k in range(3)]
    out += [("site_xpos", s, k) for s in range(m.nsite) for k in range(3)]
    return out


def element(u0, u1, step, E):
    return (int(u0) + int(step) * int(u1)) % E


# ---- probe envs ---------------------------------------------------------------------------------------
class _Probe:
    """Mixin: the probe reward, ``sweep`` = (user[0], user[1]) of e(s)."""
    reward_source = PROBE
    sweep = (0, 1)

    def user_params(self):
        return np.array(self.sweep, dtype=np.float32)

    def probed(self, u0, u1=1):
        """A copy of this env (same model and build) that reads element (u0 + s u1) mod E at step s."""
        e = copy.copy(self)
        e.sweep = (int(u0), int(u1))
        return e


def _classes():
    if EX not in sys.path:
        sys.path.insert(0, EX)
    import pincher_env
    import quadpod_env
    from dial_mpc_b200.config.base_env_config import BaseEnvConfig
    from dial_mpc_b200.envs.base_env import System
    from dial_mpc_b200.envs.custom_env import CustomRewardEnv
    from dial_mpc_b200.envs.unitree_h1_env import UnitreeH1LocoEnvConfig as H1LocoCfg
    from dial_mpc_b200.envs.unitree_h1_env import UnitreeH1WalkEnvConfig as H1Cfg
    from dial_mpc_b200.modelc import CompiledModel, compile_mjcf
    from dial_mpc_b200.utils.io_utils import get_model_path
    from tests import tree_envs

    class StockProbe(_Probe, CustomRewardEnv):
        """A stock model (its compiled JSON, as the stock env loads it) with the probe reward."""
        model = ("", "")
        ranges = None       # the stock env's sampling range of the joint targets

        def __init__(self, config):
            super().__init__(config)
            if self.ranges is not None:
                self.joint_range = np.array(self.ranges)

        def make_system(self, config):
            sys = System(CompiledModel.load(get_model_path(*self.model)))
            return sys.tree_replace({"opt.timestep": config.timestep})

    class Go2Probe(StockProbe):
        model = ("unitree_go2", "mjx_scene_force.xml")
        ranges = [[-0.5, 0.5], [0.4, 1.4], [-2.3, -0.85]] * 2 + [[-0.5, 0.5], [0.4, 1.4], [-2.3, -1.3]] * 2

    class H1WalkProbe(StockProbe):
        model = ("unitree_h1", "mjx_scene_h1_walk.xml")
        ranges = ([[-0.3, 0.3], [-0.3, 0.3], [-1.0, 1.0], [0.0, 1.74], [-0.6, 0.4]] * 2 + [[-0.5, 0.5]]
                  + [[-0.78, 0.78], [-0.3, 0.3], [-0.3, 0.3], [-0.3, 0.3]] * 2)

    class H1LocoProbe(StockProbe):
        model = ("unitree_h1", "mjx_scene_h1_loco.xml")
        ranges = [[-0.2, 0.2], [-0.2, 0.2], [-0.6, 0.6], [0.0, 1.5], [-0.6, 0.4]] * 2 + [[-0.5, 0.5]]

    class AllegroProbe(StockProbe):
        model = ("wonik_allegro", "scene_left.xml")
        init_keyframe = "in_hand_reorient"

    class SpheresProbe(_Probe, pincher_env.PincherEnv):
        def make_system(self, config):
            sys = System(compile_mjcf(os.path.join(MODELS, "spheres.xml")))
            return sys.tree_replace({"opt.timestep": config.timestep})

    def tree(cls):
        return type(cls.__name__ + "Probe", (_Probe, cls), {})

    T = tree_envs.TreeEnvConfig
    # name -> (class, config class, configuration, the solver variant the model must pick (, dense nv))
    return {
        "go2": (Go2Probe, BaseEnvConfig, dict(kp=30.0, kd=0.0), (1, None)),                 # star<3,6>
        "quadpod": (tree(quadpod_env.QuadpodEnv), quadpod_env.QuadpodEnvConfig, {}, (1, None)),
        "slidepod": (tree(tree_envs.SlidepodEnv), T, tree_envs.FIXTURES["slidepod"][1], (1, None)),
        "h1_walk": (H1WalkProbe, H1Cfg, {}, (2, None)),          # star<5,7>
        "h1_loco": (H1LocoProbe, H1LocoCfg, {}, (4, None)),          # star<5,6>
        "allegro": (AllegroProbe, BaseEnvConfig, dict(kp=1.0, kd=0.1, leg_control="position", dt=0.005,
                                                      timestep=0.005), (3, 22)),            # dense nv = 22
        "pincher": (tree(pincher_env.PincherEnv), pincher_env.PincherEnvConfig, dict(dt=0.005), (3, 10)),
        "spheres": (SpheresProbe, pincher_env.PincherEnvConfig, dict(dt=0.005), (3, 10)),
        "branchpod": (tree(tree_envs.BranchpodEnv), T, tree_envs.FIXTURES["branchpod"][1], (0, None)),
        "hexapod": (tree(tree_envs.HexapodEnv), T, tree_envs.FIXTURES["hexapod"][1], (0, None)),
        "longchain": (tree(tree_envs.LongchainEnv), T, tree_envs.FIXTURES["longchain"][1], (0, None)),
    }


NAMES = ["go2", "quadpod", "slidepod", "h1_walk", "h1_loco", "allegro", "pincher", "spheres", "branchpod",
         "hexapod", "longchain"]
_CLASSES = None


def variant_of(name):
    global _CLASSES
    if _CLASSES is None:
        _CLASSES = _classes()
    return _CLASSES[name][3]


@functools.lru_cache(maxsize=None)
def make_probe(name, **overrides):
    """(probe env, fp64 oracle model) of a probe env; ``overrides`` go into the env configuration (the
    default has one physics substep per env step)."""
    global _CLASSES
    from oracle.mjx_oracle import OModel
    if _CLASSES is None:
        _CLASSES = _classes()
    cls, cfg_cls, kw, _ = _CLASSES[name]
    cfg = cfg_cls(**dict(kw, **overrides))
    env = cls(cfg)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, name + ".json")
        env.sys.model.save(path)
        om = OModel(path)
    return env, om


def emul_defines(env):
    """Compile-time options of the CPU warp emulator for this model: the dense solver for its nv."""
    from dial_mpc_b200 import custom
    nvd = custom.dense_nv(env.sys.model)
    return (f"DIAL_DENSE_NV={nvd}",) if nvd not in (None, 22) else ()


# ---- the fp64 reference and its tolerance -------------------------------------------------------------
def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def _sincos_err(x, sfu):
    """Absolute error of the kernel's sin / cos of x: libm (emulator) or the SFU's __sincosf (GPU)."""
    return 2.0 ** -21.41 + 2 * _ulp(x) if sfu else 2 * E32 + 0 * x


def _norm(x):
    return np.linalg.norm(x, axis=-1)


def reference(om, q, qd, q_post, qd_post, sfu):
    """(ref [R, E], tol [R, E]) of every element for rows whose step started from (q, qd) [R, nq / nv] and
    ended at (q_post, qd_post).  Kinematic fields from the pre-state in fp64; qpos / qvel: the post-state,
    tolerance 0.  ``sfu``: the GPU's sin / cos error model (else the emulator's)."""
    from oracle import mjx_oracle as mo
    q, qd = np.asarray(q, np.float64), np.asarray(qd, np.float64)
    R, nb = q.shape[0], om.nbody
    qn, xpos, xquat, xmat, xipos, ximat, xanchor, xaxis = mo.kinematics(om, q)
    root_com, cinert, cdof = mo.com_pos(om, xpos, xmat, xipos, ximat, xanchor, xaxis)
    cvel, _ = mo.com_vel(om, cdof, qd)
    dist, cpos, _ = mo.collision(om, xpos, xmat)
    ang = cvel[..., :3]
    off = xpos - root_com
    vel = cvel[..., 3:] - np.cross(off, ang)
    site = xpos[:, om.site_bodyid] + np.einsum("nsij,sj->nsi", xmat[:, om.site_bodyid], om.site_pos)

    # bounds (module docstring)
    th, dx, danc = np.zeros((R, nb)), np.zeros((R, nb)), np.zeros((R, nb))
    for b in range(1, nb):
        p, j = int(om.body_parentid[b]), int(om.body_jntadr[b])
        t = th[:, p] + 8 * E32
        L = np.linalg.norm(om.body_pos[b]) + np.zeros(R)
        if j >= 0:
            qa, jt = int(om.jnt_qposadr[j]), int(om.jnt_type[j])
            if jt == mo.JNT_FREE:
                t = 8 * E32 + np.zeros(R)
            else:
                dq = q[:, qa] - om.qpos0[qa]
                L = L + 2 * np.linalg.norm(om.jnt_pos[j])
                if jt == mo.JNT_HINGE:
                    t = t + _ulp(dq) + 4 * _sincos_err(dq / 2, sfu)
                else:
                    L = L + np.abs(dq)
        th[:, b] = t
        if j >= 0 and int(om.jnt_type[j]) == mo.JNT_FREE:
            dx[:, b] = 0.0
        else:
            dx[:, b] = dx[:, p] + L * t + 4 * E32 * (_norm(xpos[:, b]) + L)
            if j >= 0 and int(om.jnt_type[j]) == mo.JNT_SLIDE:
                dx[:, b] += _ulp(q[:, int(om.jnt_qposadr[j])] - om.qpos0[int(om.jnt_qposadr[j])])
        danc[:, b] = dx[:, b] + (2 * np.linalg.norm(om.jnt_pos[j]) if j >= 0 else 0.0) * 4 * t

    def point(b, o, p_world):
        on = np.linalg.norm(o, axis=-1)
        return dx[:, b] + 4 * th[:, b] * on + 4 * E32 * (_norm(p_world) + on)

    dxi = np.stack([point(b, om.body_ipos[b], xipos[:, b]) for b in range(nb)], 1)
    dcom = np.zeros((R, nb))
    for r in np.unique(om.body_rootid):
        sel = om.body_rootid == r
        dcom[:, sel] = (dxi[:, sel].max(1) + 2 * E32 * sel.sum() * _norm(xipos[:, sel]).max(1))[:, None]
    # dial_xd_vel = cvel_lin - (x - com) x cvel_ang with cvel_lin = sum qd_j axis_j x (com - anchor_j): the kernel's
    # fp32 subtree COM enters both terms as the same value and cancels, leaving sum qd_j axis_j x (x - anchor_j)
    dang, dvel, nchain = np.zeros((R, nb)), np.zeros((R, nb)), np.zeros(nb)
    for d in range(om.nv):
        bd = int(om.dof_bodyid[d])
        j = int(om.dof_jntid[d])
        moved = om.body_dofmask[:, d]
        nchain[moved] += 1
        if int(om.jnt_type[j]) == mo.JNT_FREE and d - int(om.jnt_dofadr[j]) < 3:
            continue                                       # translational dofs of a free joint: exact unit vectors
        qa = np.abs(qd[:, d])[:, None]
        arm = _norm(xpos[:, moved] - xanchor[:, bd][:, None])
        dang[:, moved] += qa * (2 * th[:, bd] + 4 * E32)[:, None]
        dvel[:, moved] += qa * (2 * th[:, bd][:, None] * arm + dx[:, moved] + danc[:, bd][:, None]
                                + 4 * E32 * (_norm(root_com[:, bd]) + _norm(xanchor[:, bd]))[:, None])
    angn, linn, offn = _norm(ang), _norm(cvel[..., 3:]), _norm(off)
    dang = dang + 2 * E32 * nchain * angn
    dvel = dvel + (2 * E32 * nchain + 4 * E32) * (linn + offn * angn)

    # contacts
    tdist, tpos = np.zeros((R, om.ncon)), np.zeros((R, om.ncon))
    c = 0
    for k in range(om.npair):
        g1, g2 = int(om.pair_geom1[k]), int(om.pair_geom2[k])
        b1, b2 = int(om.geom_bodyid[g1]), int(om.geom_bodyid[g2])
        gp = lambda g, b: xpos[:, b] + np.einsum("nij,j->ni", xmat[:, b], om.geom_pos[g])
        p1, p2 = gp(g1, b1), gp(g2, b2)
        dg1, dg2 = point(b1, om.geom_pos[g1], p1), point(b2, om.geom_pos[g2], p2)
        r1, r2 = om.geom_size[g1, 0], om.geom_size[g2, 0]
        kind = int(om.pair_kind[k])
        if kind in (mo.PAIR_PLANE_SPHERE, mo.PAIR_PLANE_CAPSULE):
            for s in range(int(om.pair_ncon[k])):
                hl = om.geom_size[g2, 1] if kind == mo.PAIR_PLANE_CAPSULE else 0.0
                dc = dg2 + hl * (4 * th[:, b2] + 4 * E32) + 2 * E32 * (_norm(p2) + hl)
                tdist[:, c] = dc + 4 * th[:, b1] * (_norm(p2 - p1) + hl) + dg1 + 4 * E32 * (_norm(p2) + hl + _norm(p1) + r2)
                tpos[:, c] = dc + tdist[:, c] / 2 + 4 * th[:, b1] * r2 + 4 * E32 * (_norm(cpos[:, c]) + r2)
                c += 1
            continue
        hl1 = om.geom_size[g1, 1] if kind == mo.PAIR_CAPSULE_CAPSULE else 0.0
        hl2 = om.geom_size[g2, 1] if kind in (mo.PAIR_SPHERE_CAPSULE, mo.PAIR_CAPSULE_CAPSULE) else 0.0
        dq1 = dg1 + hl1 * (4 * th[:, b1] + 4 * E32) + 4 * E32 * (_norm(p1) + hl1)
        dq2 = dg2 + hl2 * (4 * th[:, b2] + 4 * E32) + 4 * E32 * (_norm(p2) + hl2)
        if kind == mo.PAIR_SPHERE_CAPSULE:
            dq2 = dq2 + dq1
        extra = 0.0
        if kind == mo.PAIR_CAPSULE_CAPSULE:
            a, bb = xmat[:, b1] @ mo.qmat(om.geom_quat[g1])[:, 2], xmat[:, b2] @ mo.qmat(om.geom_quat[g2])[:, 2]
            dd = np.sum(a * bb, -1)
            daxis = 4 * np.maximum(th[:, b1], th[:, b2]) + 4 * E32
            base = dq1 + dq2
            extra = np.minimum((2 * base + 4 * (_norm(p1 - p2) + hl1 + hl2) * daxis) / (1 - dd * dd + 1e-6),
                               2 * (hl1 + hl2))
        dn = dist[:, c] + r1 + r2            # |q2 - q1|
        ddist = dq1 + dq2 + 4 * E32 * (np.abs(dn) + r1 + r2)
        dnrm = np.where(dn == 0.0, 0.0, np.minimum(2 * (dq1 + dq2 + 2 * extra + 4 * E32 * dn) / np.maximum(dn, 1e-30), 2.0))
        tdist[:, c] = ddist
        tpos[:, c] = dq1 + extra + np.abs(r1 + dist[:, c] / 2) * dnrm + ddist / 2 + 4 * E32 * _norm(cpos[:, c])
        c += 1

    # flat, in the probe's order
    body_ref = np.concatenate([xpos, xquat, xmat.reshape(R, nb, 9), ang, vel], -1)            # [R, nb, 22]
    one = np.ones((R, nb, 1))
    body_tol = np.concatenate([dx[..., None] * np.ones(3), (2 * th + 2 * E32)[..., None] * np.ones(4),
                               (4 * th + 4 * E32)[..., None] * np.ones(9), dang[..., None] * np.ones(3),
                               dvel[..., None] * np.ones(3)], -1) * one
    sb = om.site_bodyid
    site_tol = np.stack([point(int(b), om.site_pos[s], site[:, s]) for s, b in enumerate(sb)], 1) if om.nsite else np.zeros((R, 0))
    ref = np.concatenate([np.asarray(q_post, np.float64), np.asarray(qd_post, np.float64), body_ref.reshape(R, -1),
                          np.concatenate([dist[..., None], cpos], -1).reshape(R, -1), site.reshape(R, -1)], 1)
    tol = np.concatenate([np.zeros((R, om.nq + om.nv)), body_tol.reshape(R, -1),
                          np.concatenate([tdist[..., None], tpos[..., None] * np.ones(3)], -1).reshape(R, -1),
                          (site_tol[..., None] * np.ones(3)).reshape(R, -1)], 1)
    return ref, tol


def check_elements(om, got, elems, ref, tol, what, worst=None):
    """got [R, T] of elements elems [R, T] against ref / tol [R, E] (one state per row)."""
    worst = {} if worst is None else worst
    lay = layout(om)
    got = np.asarray(got, np.float64)
    r_ = np.take_along_axis(ref, elems, 1)
    t_ = np.take_along_axis(tol, elems, 1)
    err = np.abs(got - r_)
    assert np.isfinite(got).all(), f"{what}: non-finite value read"
    exact = t_ == 0
    bad = exact & (err != 0)
    assert not bad.any(), f"{what}: {lay[int(elems[bad][0])]} differs from its exact value: " \
                          f"{got[bad][0]!r} vs {r_[bad][0]!r}"
    ratio = np.where(exact, 0.0, err / np.where(exact, 1.0, t_))
    i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    assert ratio.max() <= 1.0, (f"{what}: {lay[int(elems[i])]}: got {got[i]!r}, fp64 {r_[i]!r}, "
                                f"tol {t_[i]:.3g} ({ratio[i]:.3g} x)")
    for f in set(lay[int(x)][0] for x in np.unique(elems)):
        sel = np.vectorize(lambda x: lay[int(x)][0] == f)(elems)
        worst[f] = max(worst.get(f, 0.0), float(ratio[sel].max()))
    return worst


def fields_of(om):
    """The fields of the contract this model exposes (contacts and sites if it has any)."""
    f = {"qpos", "qvel"} | {n for n, _ in BODY_FIELDS}
    if om.ncon:
        f |= {"contact_dist", "contact_pos"}
    if om.nsite:
        f |= {"site_xpos"}
    return f


def ref_steps(om, rows_q, rows_qd, q0, qd0, sfu):
    """ref / tol [R, H, E] of every step of rollouts that started from (q0, qd0) and stored
    rows_q [R, H, nq], rows_qd [R, H, nv]."""
    R, H = rows_q.shape[:2]
    pre_q = np.concatenate([np.repeat(np.asarray(q0, np.float64)[None, None], R, 0), rows_q[:, :-1]], 1)
    pre_qd = np.concatenate([np.repeat(np.asarray(qd0, np.float64)[None, None], R, 0), rows_qd[:, :-1]], 1)
    ref, tol = reference(om, pre_q.reshape(R * H, -1), pre_qd.reshape(R * H, -1), rows_q.reshape(R * H, -1),
                         rows_qd.reshape(R * H, -1), sfu)
    return ref.reshape(R, H, -1), tol.reshape(R, H, -1)


# ---- states ---------------------------------------------------------------------------------------------
def actions(env, R, H, seed, scale=1.0):
    return np.clip(np.random.default_rng(seed).standard_normal((R, H, env.action_size)) * scale, -1, 1).astype(np.float32)


def lifted(env, dz, seed):
    """The env's initial pose raised by dz, with a tilted root and random velocities: far from the ground."""
    g = np.random.default_rng(seed)
    q = np.asarray(env._init_q, np.float64).copy()
    qd = 0.5 * g.standard_normal(env.sys.nv)
    if env.sys.model.jnt_type[0] == 0:
        q[2] += dz
        quat = q[3:7] + 0.3 * g.standard_normal(4)
        q[3:7] = quat / np.linalg.norm(quat)
    return q.astype(np.float32), qd.astype(np.float32)


def edge_states(name, env, om):
    """Constructed start states at the edges of the kinematics and the contacts: [(label, qpos, qvel)]."""
    m = env.sys.model
    q0 = np.asarray(env._init_q, np.float64)
    g = np.random.default_rng(len(name))
    out = []
    free = m.jnt_type[0] == 0
    qd = (0.3 * g.standard_normal(m.nv))
    if free:
        for label, quat in (("quat identity", [1, 0, 0, 0]), ("quat 180 deg", [0, 0.6, 0.8, 0]),
                            ("quat x 1e-2", 1e-2 * np.array([0.9, 0.1, -0.3, 0.3])),
                            ("quat x 10", 10 * np.array([0.5, -0.5, 0.5, 0.5]))):
            q = q0.copy()
            q[3:7] = quat
            out.append((label, q, qd))
    hinge = [j for j in range(m.njnt) if m.jnt_type[j] == 3]
    lo = np.array([m.jnt_range[j, 0] for j in hinge])
    hi = np.array([m.jnt_range[j, 1] for j in hinge])
    qa = np.array([m.jnt_qposadr[j] for j in hinge], int)
    if len(hinge):
        for label, vals in (("hinges at lower limits", lo), ("hinges at upper limits", hi),
                            ("hinges beyond limits", hi + 1.5), ("hinges wound past 2 pi", q0[qa] + 7.0),
                            ("hinges wound past -4 pi", q0[qa] - 13.0)):
            q = q0.copy()
            q[qa] = vals
            out.append((label, q, qd))
    return out


def touching(env, om, pair_kind, depth):
    """The root placed so that the lowest geom of a pair of kind ``pair_kind`` with the plane is at distance
    -depth (0: exactly touching), from the initial pose; None if no such pair."""
    from oracle import mjx_oracle as mo
    m = env.sys.model
    q = np.asarray(env._init_q, np.float64).copy()
    if m.jnt_type[0] != 0:
        return None
    ks = [k for k in range(om.npair) if om.pair_kind[k] == pair_kind]
    if not ks:
        return None
    d, *_ = mo.collision(om, *mo.kinematics(om, q[None])[1:4:2])
    cons = [c for c in range(om.ncon) if om.con_pair[c] in ks]
    lowest = min(cons, key=lambda c: d[0, c])
    q[2] -= d[0, lowest] + depth
    # an fp32-exact touching height: the distance of the fp32 state is recomputed by the caller's reference
    return q.astype(np.float32)


# ---- runs ---------------------------------------------------------------------------------------------
def sweep_stride(E, prefer=(1,)):
    """The first stride of ``prefer`` coprime with E (then 7, 11, 13, ...): a sweep with it reads every element."""
    import math
    return next(s for s in tuple(prefer) + (7, 11, 13, 17, 19, 23) if math.gcd(s, E) == 1)


def sweep_starts(E, H, u1=1):
    """u0 of the ceil(E / H) launches of H steps with stride u1 (coprime with E) that together read every element:
    launch l reads u1 (l H + t) mod E at step t."""
    return [(u1 * l * H) % E for l in range(-(-E // H))]


def edge_elements(om, rng, n=12):
    """The elements read at t = 0 of an edge state: the first root body's xquat, the deepest body's xpos and
    xquat, one element of every field of every contact, and a random sample of n others."""
    lay = layout(om)
    deep = int(np.argmax(om.body_dofmask.sum(1)))
    keep = [i for i, f in enumerate(lay) if (f[0] == "xquat" and f[1] in (1, deep)) or (f[0] == "xpos" and f[1] == deep)
            or f[0] == "contact_dist" or (f[0] == "contact_pos" and f[2] == 2)]
    return sorted(set(keep) | set(rng.choice(len(lay), n, replace=False).tolist()))


def preroll(launch, env, q0, qd0, steps, seed, H=32):
    """The state row 0 of chained random-action launches reaches after ``steps`` env steps from (q0, qd0): a
    mid-rollout state, contacts made and broken on the way."""
    q, qd = np.asarray(q0, np.float32), np.asarray(qd0, np.float32)
    for k in range(-(-steps // H)):
        _, qs, qds = launch(q, qd, actions(env, 1, H, seed + k, 0.7), 0, 1)
        q, qd = np.asarray(qs[0, -1], np.float32), np.asarray(qds[0, -1], np.float32)
    return q, qd


def emul_launch(env, q0, qd0, us, u0, u1=1):
    """(rewss [R, H], q [R, H, nq], qd [R, H, nv]) of the CPU warp emulator: one launch of explicit actions."""
    from tests.emul import emul
    out = emul.rollout(env.probed(u0, u1), env.probed(u0, u1).plan_desc(), q0, qd0, np.zeros(env.sys.nv, np.float32),
                       us=us, defines=emul_defines(env))
    return out["rewss"], out["q"], out["qd"]


def run_checks(om, launch, q0, qd0, us, starts, sfu, what, worst=None, u1=1):
    """Launch once per u0 in ``starts`` from (q0, qd0) with actions us [R, H, nu]; every value read against fp64.
    ``launch(q0, qd0, us, u0, u1)`` -> (rewss, q, qd).  Returns {field: worst ratio} and the elements read."""
    E = n_elements(om)
    worst = {} if worst is None else worst
    seen = set()
    for u0 in starts:
        rewss, q, qd = launch(q0, qd0, us, u0, u1)
        R, H = rewss.shape
        ref, tol = ref_steps(om, np.asarray(q, np.float64), np.asarray(qd, np.float64), q0, qd0, sfu)
        el = np.array([element(u0, u1, t, E) for t in range(H)])
        check_elements(om, rewss.reshape(R * H, 1), np.repeat(el[None], R, 0).reshape(R * H, 1),
                       ref.reshape(R * H, -1), tol.reshape(R * H, -1), f"{what} u0={u0}", worst)
        seen |= set(el.tolist())
    return worst, seen


def pitched(env, angle=np.pi / 2):
    """The initial pose with the free root pitched by ``angle`` about y: capsules along x stand on their axis."""
    q = np.asarray(env._init_q, np.float64).copy()
    if env.sys.model.jnt_type[0] != 0:
        return None
    q[3:7] = [np.cos(angle / 2), 0.0, np.sin(angle / 2), 0.0]
    return q


def coincident_spheres(env):
    """spheres.xml: the ball centred on the left tip sphere at zero hinge angles (both centres exact in fp32)."""
    q = np.zeros(env.sys.nq)
    q[0:3] = [-0.03125, 0.0, 0.015625]
    q[3] = 1.0
    return q


def cc_conditioning(om, q):
    """min over the capsule-capsule pairs of 1 - (a.b)^2 at the states q [R, nq] (inf if none)."""
    from oracle import mjx_oracle as mo
    _, xpos, _, xmat, *_ = mo.kinematics(om, np.asarray(q, np.float64))
    out = np.inf
    for k in range(om.npair):
        if om.pair_kind[k] != mo.PAIR_CAPSULE_CAPSULE:
            continue
        g1, g2 = int(om.pair_geom1[k]), int(om.pair_geom2[k])
        a = xmat[:, om.geom_bodyid[g1]] @ mo.qmat(om.geom_quat[g1])[:, 2]
        b = xmat[:, om.geom_bodyid[g2]] @ mo.qmat(om.geom_quat[g2])[:, 2]
        out = min(out, float((1 - np.sum(a * b, -1) ** 2).min()))
    return out
