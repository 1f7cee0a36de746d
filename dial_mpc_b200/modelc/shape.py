"""Integer structure of a compiled model as the ``-DDIAL_SHAPE_*`` defines of a specialised rollout kernel
(``ShapeFixed`` in csrc/dial_device.cuh).

The stock library builds the star<3,6> kernel once more for each entry of ``SHAPES``, specialised on the
values derived here from the model JSON the environment loads: body / dof / actuator counts, tree depth,
kinematic trees, the star chains, the contact pair kind, the contact and pyramid-edge counts and the
solver's iteration counts; and from the environment's plan under its default configuration: the number of
feet and the physics steps per env step.  A plan uses such a kernel only when the host finds every one of
these values equal to its own model and plan (``shape_matches``); anything else runs the generic kernel.
Float data (masses, time steps, gains, ranges) is never part of the structure."""
from __future__ import annotations

from typing import List, Optional

# (kernel name, environment that loads the model): the Go2 scene (models/unitree_go2_mjx_scene_force.json),
# shared by the walk and jump envs
SHAPES = (("go2", "unitree_go2_walk"),)


def structure_defines(md, pd=None) -> Optional[List[str]]:
    """``NAME=value`` defines of the structure of model descriptor ``md`` (and, given plan descriptor
    ``pd``, of the plan's feet and physics steps per env step), or None when it has no single value for a
    field the policy fixes (chains of different lengths, mixed contact pair kinds, no star of hanging
    chains)."""
    nb, nv = md.nbody, md.nv
    depth = [md.body_depth[b] for b in range(1, nb)]
    roots = {md.body_rootid[b] for b in range(1, nb)}
    # star chains as the host derives them (dial_host.h derive_star): from every leaf dof up while the
    # dofs have at most one child; the remaining dofs form the root chain
    nchild = [0] * nv
    for i in range(nv):
        if md.dof_parentid[i] >= 0:
            nchild[md.dof_parentid[i]] += 1
    inchain, lens = [False] * nv, []
    for i in range(nv):
        if nchild[i]:
            continue
        n, j = 0, i
        while j >= 0 and nchild[j] <= 1:
            inchain[j] = True
            n += 1
            j = md.dof_parentid[j]
        lens.append(n)
    root_dofs = [i for i in range(nv) if not inchain[i]]
    root_bodies = []
    for d in reversed(root_dofs):            # deepest first, one entry per body
        b = md.dof_bodyid[d]
        if not root_bodies or root_bodies[-1] != b:
            root_bodies.append(b)
    kinds = {md.pair_kind[k] for k in range(md.npair) if md.pair_ncon[k] > 0}
    if not lens or len(set(lens)) != 1 or len(kinds) != 1 or not root_dofs:
        return None
    vals = dict(NBODY=nb, NQ=md.nq, NV=nv, NU=md.nu, MAXDEPTH=max(depth), NROOT=len(roots), NCHAIN=len(lens),
                CHAINLEN=lens[0], SB_NROOT=len(root_bodies), PAIR_KIND=kinds.pop(), ITERATIONS=md.iterations,
                LS_ITERATIONS=md.ls_iterations,
                # pyramidal cones: four edges per contact (dial_host.h, DevModel.nedge of the star paths)
                NCON=md.ncon, NEDGE=4 * md.ncon)
    if pd is not None:
        vals.update(NFEET=pd.nfeet, N_FRAMES=pd.n_frames)
    return [f"DIAL_SHAPE_{k}={int(v)}" for k, v in vals.items()]


def env_structure_defines(env_name: str) -> List[str]:
    """The defines of the model a registered environment loads, and of its plan, under its default
    configuration."""
    import dial_mpc_b200.envs as E
    from dial_mpc_b200 import _capi
    env = E.get_environment(env_name, config=E.get_config(env_name)())
    d = structure_defines(_capi.fill_model_desc(env.sys.model), env.plan_desc())
    if d is None:
        raise ValueError(f"{env_name}: the model has no fixed structure to specialise on")
    return d
