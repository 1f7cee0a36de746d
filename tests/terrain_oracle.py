"""TEST-ONLY: the per-instance terrain (dial_mpc_b200/terrain.py, include/dial_b200.h) restated in fp64 on top of
the oracle: the floor contacts of ``mjx_oracle.collision`` measured against the plane of the terrain's triangle
under each sphere (or capsule end), and the built-in rewards' terrain-relative height terms.  The surface is
restated here from the definition (include/dial_b200.h), not taken from the library's Python."""
import contextlib

import numpy as np

import oracle.envs_oracle as eo
import oracle.mjx_oracle as mo


def plane(t, x, y):
    """(H, sx, sy) of terrain t under the world points (x, y) in fp64: the vertices of the triangle under the point
    (the cell's diagonal runs from (i, j) to (i+1, j+1)), the plane through them, evaluated at the point; outside
    the grid, the height of the point clamped into it and slopes 0."""
    h = np.asarray(t.heights, dtype=np.float64)
    ny, nx = h.shape
    s = float(t.spacing)
    gx = (np.asarray(x, dtype=np.float64) - t.origin[0]) / s
    gy = (np.asarray(y, dtype=np.float64) - t.origin[1]) / s
    out = (gx < 0) | (gx > nx - 1) | (gy < 0) | (gy > ny - 1)
    gx, gy = np.clip(gx, 0, nx - 1), np.clip(gy, 0, ny - 1)
    i = np.clip(np.floor(gx).astype(np.int64), 0, nx - 2)
    j = np.clip(np.floor(gy).astype(np.int64), 0, ny - 2)
    # triangle vertices in grid units: (0, 0), (1, 1) and (1, 0) below the diagonal, (0, 1) above it
    below = gx - i >= gy - j
    p0 = np.stack([i, j, h[j, i]], -1).astype(np.float64)
    p1 = np.stack([i + 1, j + 1, h[j + 1, i + 1]], -1).astype(np.float64)
    p2 = np.where(below[..., None], np.stack([i + 1, j, h[j, i + 1]], -1), np.stack([i, j + 1, h[j + 1, i]], -1))
    nrm = np.cross(p1 - p0, p2 - p0)                    # the plane's normal in grid units (x, y) and metres (z)
    dzdx, dzdy = -nrm[..., 0] / nrm[..., 2], -nrm[..., 1] / nrm[..., 2]
    H = p0[..., 2] + dzdx * (gx - p0[..., 0]) + dzdy * (gy - p0[..., 1])
    return H, np.where(out, 0.0, dzdx / s), np.where(out, 0.0, dzdy / s)

_floor_collision = mo.collision   # (on_terrain replaces mo.collision, which forward() calls)


def floor_pairs(m):
    """Contact slots of the floor pairs (plane-sphere / plane-capsule with the plane on the world body), in the
    order of ``mjx_oracle.collision``: [(slot, pair, capsule end sign or 0)]."""
    out, c = [], 0
    for k in range(m.npair):
        kind = int(m.pair_kind[k])
        floor = kind in (mo.PAIR_PLANE_SPHERE, mo.PAIR_PLANE_CAPSULE) and int(m.geom_bodyid[int(m.pair_geom1[k])]) == 0
        ends = (1.0, -1.0) if kind == mo.PAIR_PLANE_CAPSULE else (0.0,)
        for sgn in ends:
            if floor:
                out.append((c, k, sgn))
            c += 1
    return out


def collision(m, xpos, xmat, t):
    """``mjx_oracle.collision`` with the floor pairs on terrain ``t`` (None: the floor)."""
    dist, pos, frame = _floor_collision(m, xpos, xmat)
    if t is None:
        return dist, pos, frame
    for c, k, sgn in floor_pairs(m):
        g2 = int(m.pair_geom2[k])
        b2 = int(m.geom_bodyid[g2])
        p2 = xpos[:, b2] + np.einsum("nij,j->ni", xmat[:, b2], m.geom_pos[g2])
        R2 = np.einsum("nij,jk->nik", xmat[:, b2], mo.qmat(m.geom_quat[g2]))
        r = m.geom_size[g2, 0]
        cc = p2 + sgn * R2[:, :, 2] * m.geom_size[g2, 1]
        H, sx, sy = plane(t, cc[:, 0], cc[:, 1])
        n = np.stack([-sx, -sy, np.ones_like(sx)], -1)
        n = n / np.linalg.norm(n, axis=-1, keepdims=True)
        o = np.stack([cc[:, 0], cc[:, 1], H], -1)
        d = np.sum((cc - o) * n, -1) - r
        dist[:, c] = d
        pos[:, c] = cc - n * (r + 0.5 * d)[:, None]
        if sgn == 0.0:
            frame[:, c] = mo.make_frame(n)
        else:   # the plane-capsule frame of mjx_oracle.collision with this end's normal
            axis = R2[:, :, 2]
            bvec = axis - n * np.sum(n * axis, -1, keepdims=True)
            bn = np.linalg.norm(bvec, axis=-1, keepdims=True)
            bdir = bvec / (bn + 1e-6 * (bn == 0.0))
            alt = np.where(((n[:, 1] > -0.5) & (n[:, 1] < 0.5))[:, None], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0])
            bdir = np.where(bn < 0.5, alt, bdir)
            frame[:, c] = np.stack([n, bdir, np.cross(n, bdir)], axis=-2)
    return dist, pos, frame


def height_terms(o, s, d, t):
    """The change the terrain makes to o's reward for the step s -> d: the base height (Go2 walk, H1 walk, H1 loco)
    and Go2 walk's foot heights measured above the terrain beneath instead of above z = 0."""
    if t is None or isinstance(o, eo.Go2SeqJumpOracle) or not isinstance(o, (eo.Go2WalkOracle, eo.H1WalkOracle)):
        return 0.0
    base = d.xpos[:, o.torso + 1]
    zt = o.pos_tar[2]
    hb = plane(t, base[:, 0], base[:, 1])[0]
    delta = (0.5 if isinstance(o, eo.H1WalkOracle) else 1.0) * ((base[:, 2] - zt) ** 2 - (base[:, 2] - hb - zt) ** 2)
    if isinstance(o, eo.Go2WalkOracle):
        feet = d.site_xpos[:, o.feet_site]
        hf = plane(t, feet[..., 0], feet[..., 1])[0]
        duty, cad, amp = o.GAIT_PARAMS[o.gait]
        z_tar = eo.get_foot_step(duty, cad, amp, o.GAIT_PHASE[o.gait], s.step.astype(np.float64) * o.dt)
        delta = delta + 0.1 * (np.sum(((z_tar - feet[..., 2]) / 0.05) ** 2, -1)
                               - np.sum(((z_tar - feet[..., 2] + hf) / 0.05) ** 2, -1))
    return delta


@contextlib.contextmanager
def on_terrain(o, t):
    """The oracle env o with its physics and reward on terrain t (restored on exit)."""
    reward = o.reward
    mo.collision = lambda m, xpos, xmat: collision(m, xpos, xmat, t)

    def rew(s, qpos, qvel, d, ctrl):
        r, stage = reward(s, qpos, qvel, d, ctrl)
        return r + height_terms(o, s, d, t), stage
    o.reward = rew
    try:
        yield o
    finally:
        mo.collision = _floor_collision
        del o.reward
