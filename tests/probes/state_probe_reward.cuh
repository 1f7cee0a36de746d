// TEST-ONLY probe reward (contract: include/dial_custom_reward.h): one element of the physics state the
// reward sees.
//
// At env step s (c->step) the reward is element e = (user[0] + s * user[1]) mod E of the flat order
//   qpos[nq], qvel[nv],
//   per body b = 0 .. nbody-1 (the world included): xpos[3], xquat[4], xmat[9], dial_xd_ang[3], dial_xd_vel[3],
//   per contact: contact_dist, contact_pos[3],
//   per site: dial_site_xpos[3],
// E = nq + nv + 22 nbody + 4 ncon + 3 nsite (tests/state_probe.py restates the order).  The value is returned
// as the kernel holds it, bit for bit; the velocity and site helpers are called as a reward author calls them.
DIAL_REWARD_FN float dial_custom_reward(const dial_reward_ctx* c) {
  const int E = c->nq + c->nv + 22 * c->nbody + 4 * c->ncon + 3 * c->nsite;
  int e = (int)(((long long)c->user[0] + (long long)c->step * (long long)c->user[1]) % E);
  if (e < c->nq) return c->qpos[e];
  e -= c->nq;
  if (e < c->nv) return c->qvel[e];
  e -= c->nv;
  float v[3];
  if (e < 22 * c->nbody) {
    const int b = e / 22, k = e % 22;
    if (k < 3) return c->xpos[3 * b + k];
    if (k < 7) return c->xquat[4 * b + k - 3];
    if (k < 16) return c->xmat[9 * b + k - 7];
    if (k < 19) { dial_xd_ang(c, b, v); return v[k - 16]; }
    dial_xd_vel(c, b, v);
    return v[k - 19];
  }
  e -= 22 * c->nbody;
  if (e < 4 * c->ncon) return (e % 4 == 0) ? c->contact_dist[e / 4] : c->contact_pos[3 * (e / 4) + e % 4 - 1];
  e -= 4 * c->ncon;
  dial_site_xpos(c, e / 3, v);
  return v[e % 3];
}
