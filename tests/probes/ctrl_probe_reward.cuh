// TEST-ONLY probe reward (contract: include/dial_custom_reward.h): the control the rollout applied.
//
// user[0] = env step t, user[1] = actuator a.  The reward is ctrl[a] at step t and exactly 0 at every
// other step, so a row's reward sum is that control, bitwise, and its mean reward ctrl / H.  The reward
// runs after the physics substeps of the step; ctrl is what they applied (physics does not write it).
DIAL_REWARD_FN float dial_custom_reward(const dial_reward_ctx* c) {
  return c->step == (int)c->user[0] ? c->ctrl[(int)c->user[1]] : 0.f;
}
