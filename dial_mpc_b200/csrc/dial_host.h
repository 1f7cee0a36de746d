// dial_host.h — host-side derivation of the device model (schedules + smem layout).
// Pure C++ (no CUDA runtime) so that the test-only warp emulator can share it.
#pragma once
#include <string.h>
#include <string>
#include "dial_device.cuh"

// threads per CTA the rollout kernel is compiled for (__launch_bounds__): 512 -> 128 registers per
// thread, 448 -> 144.  The launch policy never asks for more than DIAL_MAXTHREADS / 32 warps.
#ifndef DIAL_MAXTHREADS
#define DIAL_MAXTHREADS 512
#endif
// number of dofs the dense (elliptic-cone) solver is instantiated for: its matrix rows live in registers,
// unrolled at compile time.  The stock library carries nv = 22 (Allegro hand + ball); a custom build
// (dial_mpc_b200.custom) is compiled for the dof count of its own model.
#ifndef DIAL_DENSE_NV
#define DIAL_DENSE_NV 22
#endif
static_assert(DIAL_DENSE_NV >= 1 && DIAL_DENSE_NV <= 32, "the dense solver keeps one matrix row per lane");

// Star decomposition: hanging chains = maximal serial chains ending at leaf dofs whose dofs
// all have <= 1 child; the remaining dofs must form one chain from dof 0 (the root block).
static inline void derive_star(const dial_model_desc& m, DevModel& D) {
  const int nv = m.nv;
  D.star_nroot = D.star_nchain = D.star_maxlen = 0;
  int nchild[DIAL_MAXV] = {0};
  for (int i = 0; i < nv; ++i) if (m.dof_parentid[i] >= 0) nchild[m.dof_parentid[i]]++;
  bool inchain[DIAL_MAXV] = {false};
  int nchain = 0, len[4], leaf[4], top[4];
  for (int i = 0; i < nv; ++i) {
    if (nchild[i] != 0) continue;             // leaf dof
    int l = 0, j = i, t = i;
    while (j >= 0 && nchild[j] <= 1) { inchain[j] = true; t = j; ++l; j = m.dof_parentid[j]; }
    if (nchain >= 4) return;
    len[nchain] = l; leaf[nchain] = i; top[nchain] = t; ++nchain;
  }
  // root block: the remaining dofs, must be a chain ending at dof `rl` (deepest root dof)
  int nroot = 0, rl = -1;
  for (int i = 0; i < nv; ++i) if (!inchain[i]) { ++nroot; rl = i; }
  if (nroot == 0) {
    // a single serial chain (or forest of chains): treat the top of chain 0 ... not a star
    return;
  }
  if (nroot > 8 || D.dof_nchain[rl] != nroot) return;   // root dofs must all be ancestors of rl
  for (int a = 0; a < nroot; ++a) if (inchain[D.chain_tab[rl][a]]) return;
  for (int l = 0; l < nchain; ++l) {
    int par = m.dof_parentid[top[l]], att = nroot;        // no coupling if the chain hangs off the world
    if (par >= 0) {
      att = -1;
      for (int a = 0; a < nroot; ++a) if (D.chain_tab[rl][a] == par) att = a;
      if (att < 0) return;
    }
    D.star_len[l] = len[l]; D.star_leaf[l] = leaf[l]; D.star_att[l] = att;
    D.star_maxlen = len[l] > D.star_maxlen ? len[l] : D.star_maxlen;
  }
  for (int a = 0; a < nroot; ++a) D.star_root[a] = D.chain_tab[rl][a];
  D.star_nroot = nroot; D.star_nchain = nchain;
}

// which solver instantiation fits the model: 1 = star<3,6>, 2 = star<5,7>, 4 = star<5,6>, 0 = generic tree
static inline int star_variant(const DevModel& D);

// Star layout tables (see DevModel): only for models that map to a star instantiation and whose
// contact bodies are each moved by the root chain plus at most one hanging chain.
static inline void derive_star_layout(const dial_model_desc& m, DevModel& D) {
  D.s_on = 0;
  if (D.dense) return;
  const int v = star_variant(D);
  if (v != 1 && v != 2 && v != 4) return;
  const int NL = v == 1 ? 3 : 5, NR = v == 2 ? 7 : 6;
  D.s_nrp = (NR + 3) & ~3; D.s_cs = (NL + 3) & ~3; D.s_rs = D.s_nrp + D.s_cs;
  D.s_npos = D.s_nrp + 4 * D.s_cs;
  for (int i = 0; i < m.nv; ++i) { D.s_pos[i] = 0; D.s_chain[i] = -1; D.s_depth[i] = 0; }
  for (int a = 0; a < D.star_nroot; ++a) { const int d = D.star_root[a]; D.s_pos[d] = a; D.s_chain[d] = -1; D.s_depth[d] = a; }
  for (int l = 0; l < D.star_nchain; ++l) {
    const int len = D.star_len[l], leaf = D.star_leaf[l];
    const int top = D.chain_tab[leaf][len - 1];
    if (top + len - 1 != leaf) return;              // chain dofs must be contiguous (depth-first order)
    D.s_top[l] = top;
    for (int q = 0; q < len; ++q) { D.s_pos[top + q] = D.s_nrp + l * D.s_cs + q; D.s_chain[top + q] = l; D.s_depth[top + q] = q; }
  }
  for (int c = 0; c < m.ncon; ++c) {
    const int last = D.con_lastdof[c];
    D.s_con_chain[c] = D.s_chain[last];           // -1: the body hangs off the root chain itself
  }
  D.s_on = 1;
  // body-level star (subtree sums): every non-world body is a root body or lies on one chain run
  D.sb_on = 0;
  bool covered[DIAL_MAXB] = {false};
  D.sb_nroot = 0;
  for (int a = 0; a < D.star_nroot; ++a) {             // deepest root dof first
    const int b = m.dof_bodyid[D.star_root[a]];
    if (D.sb_nroot == 0 || D.sb_root[D.sb_nroot - 1] != b) {
      if (D.sb_nroot >= 4) return;
      D.sb_root[D.sb_nroot++] = b;
      covered[b] = true;
    }
  }
  for (int r = 0; r + 1 < D.sb_nroot; ++r)
    if (m.body_parentid[D.sb_root[r]] != D.sb_root[r + 1]) return;   // root bodies must form a chain
  for (int l = 0; l < D.star_nchain; ++l) {
    const int top = m.dof_bodyid[D.s_top[l]], len = D.star_len[l];
    for (int q = 0; q < len; ++q) {
      if (m.dof_bodyid[D.s_top[l] + q] != top + q) return;          // one body per chain dof, contiguous
      if (q > 0 && m.body_parentid[top + q] != top + q - 1) return;
      covered[top + q] = true;
    }
    D.sb_top[l] = top; D.sb_len[l] = len; D.sb_att[l] = -1;
    for (int r = 0; r < D.sb_nroot; ++r) if (m.body_parentid[top] == D.sb_root[r]) D.sb_att[l] = r;
    if (D.sb_att[l] < 0 && m.body_parentid[top] != 0) return;
  }
  for (int b = 1; b < m.nbody; ++b) if (!covered[b]) return;
  D.sb_on = 1;
}

static inline bool derive_model(const dial_model_desc& m, DevModel& D, std::string& err) {
  memset(&D, 0, sizeof(D));
  D.m = m;
  const int nb = m.nbody, nv = m.nv;
  if (nb < 2 || nb > DIAL_MAXB || nv > DIAL_MAXV || m.nq > DIAL_MAXQ || m.nu > DIAL_MAXU ||
      m.ngeom > DIAL_MAXG || m.npair > DIAL_MAXP || m.ncon > DIAL_MAXC || m.nsite > DIAL_MAXS) {
    err = "model exceeds the fixed device capacities (DIAL_MAX*)";
    return false;
  }
  // dense / elliptic path: elliptic cones (contacts may then couple two moving bodies, condim 1/3/6)
  D.dense = m.cone == 1 ? 1 : 0;
  bool any_damp = false;
  for (int d = 0; d < nv; ++d) any_damp |= m.dof_damping[d] != 0.f;
  if (!D.dense && m.eulerdamp && any_damp) {
    err = "implicit Euler damping (eulerdamp) is only supported on the dense (elliptic) solver path";
    return false;
  }
  if (!D.dense && 4 * m.ncon > DIAL_MAXE) { err = "too many pyramidal contact edges"; return false; }
  // depth / children / roots
  D.maxdepth = 0;
  for (int b = 1; b < nb; ++b) D.maxdepth = m.body_depth[b] > D.maxdepth ? m.body_depth[b] : D.maxdepth;
  for (int b = 1; b < nb; ++b) {
    int nd = 0;
    for (int c = b + 1; c < nb; ++c) {
      int a = c;
      while (a > 0 && a != b) a = m.body_parentid[a];
      if (a == b) ++nd;
    }
    D.body_ndesc[b] = nd;
    for (int c = b + 1; c <= b + nd; ++c) {
      int a = c;
      while (a > 0 && a != b) a = m.body_parentid[a];
      if (a != b) { err = "bodies are not in depth-first order"; return false; }
    }
  }
  D.nroot = 0;
  for (int b = 1; b < nb; ++b) {
    int r = m.body_rootid[b], idx = -1;
    for (int i = 0; i < D.nroot; ++i) if (D.root_body[i] == r) idx = i;
    if (idx < 0) {
      if (D.nroot >= 4) { err = "more than 4 kinematic trees"; return false; }
      idx = D.nroot++;
      D.root_body[idx] = r;
    }
    D.body_rootidx[b] = idx;
  }
  for (int i = 0; i < D.nroot; ++i) {
    double mass = 0;
    for (int b = 1; b < nb; ++b) if (D.body_rootidx[b] == i) mass += m.body_mass[b];
    if (mass < 1e-15) { err = "massless kinematic tree"; return false; }
    D.root_invmass[i] = (float)(1.0 / mass);
  }
  // dof ancestor masks, chain length check, elimination levels
  for (int i = 0; i < nv; ++i) {
    uint32_t mask = 0;
    int j = i, n = 0;
    while (j >= 0) { mask |= 1u << j; j = m.dof_parentid[j]; ++n; }
    if (n > DIAL_MAXCHAIN) { err = "dof ancestor chain longer than DIAL_MAXCHAIN"; return false; }
    D.dof_ancmask[i] = mask;
    D.dof_nchain[i] = n;
    j = i; n = 0;
    while (j >= 0) { D.chain_tab[i][n++] = j; j = m.dof_parentid[j]; }
  }
  for (int i = 0; i < nv; ++i) {
    int nd = 0;
    for (int k = i + 1; k < nv; ++k) if ((D.dof_ancmask[k] >> i) & 1u) ++nd;
    D.dof_ndesc[i] = nd;
    for (int k = i + 1; k <= i + nd; ++k)
      if (!((D.dof_ancmask[k] >> i) & 1u)) { err = "dofs are not in depth-first order"; return false; }
  }
  for (int i = nv - 1; i >= 0; --i) {
    int lv = 0;
    for (int k = i + 1; k < nv; ++k)
      if (m.dof_parentid[k] == i) lv = D.dof_level[k] + 1 > lv ? D.dof_level[k] + 1 : lv;
    D.dof_level[i] = lv;
    D.nlevel = lv + 1 > D.nlevel ? lv + 1 : D.nlevel;
  }
  if (D.nlevel > DIAL_MAXLEVEL) { err = "too many elimination levels"; return false; }
  int pos = 0;
  for (int lv = 0; lv < D.nlevel; ++lv) {
    D.level_adr[lv] = pos;
    for (int i = 0; i < nv; ++i) if (D.dof_level[i] == lv) D.level_dofs[pos++] = i;
  }
  D.level_adr[D.nlevel] = pos;
  for (int b = 0; b < nb; ++b) {
    uint32_t mask = 0;
    int bb = b;
    while (bb > 0) {
      if (m.body_jntadr[bb] >= 0)
        for (int k = 0; k < m.body_dofnum[bb]; ++k) mask |= 1u << (m.body_dofadr[bb] + k);
      bb = m.body_parentid[bb];
    }
    D.body_dofmask[b] = mask;
  }
  for (int d = 0; d < nv; ++d) {
    D.dof_actuator[d] = -1;
    for (int a = 0; a < m.nu; ++a) if (m.actuator_dofadr[a] == d) D.dof_actuator[d] = a;
    int j = m.dof_jntid[d];
    D.dof_limited[d] = (m.jnt_limited[j] && m.jnt_type[j] != JNT_FREE) ? j : -1;
    if (D.dof_limited[d] >= 0) D.nlimited++;
  }
  int c = 0;
  for (int k = 0; k < m.npair; ++k) {
    const int b1 = m.geom_bodyid[m.pair_geom1[k]], b2 = m.geom_bodyid[m.pair_geom2[k]];
    if (D.dense) {
      if (m.pair_kind[k] < PAIR_PLANE_SPHERE || m.pair_kind[k] > PAIR_CAPSULE_CAPSULE) { err = "unsupported contact pair kind"; return false; }
      if (m.pair_condim[k] != 1 && m.pair_condim[k] != 3 && m.pair_condim[k] != 6) { err = "condim must be 1, 3 or 6"; return false; }
      for (int s = 0; s < m.pair_ncon[k]; ++s) {
        D.con_pair[c] = k; D.con_sub[c] = s; D.con_lastdof[c] = 0;
        D.con_dim[c] = m.pair_condim[k]; D.con_row0[c] = D.nrow_c; D.nrow_c += m.pair_condim[k];
        // packed columns of this contact's rows: the dofs that move exactly one of the two bodies
        int ncol = 0;
        for (int d = 0; d < DIAL_MAXV; ++d) {
          const bool nz = d < nv && (((D.body_dofmask[b1] >> d) & 1u) != ((D.body_dofmask[b2] >> d) & 1u));
          D.con_colidx[c][d] = nz ? (int8_t)ncol++ : (int8_t)-1;
        }
        if (ncol > D.jd_stride) D.jd_stride = ncol;
        ++c;
      }
      continue;
    }
    if (m.pair_kind[k] != PAIR_PLANE_SPHERE && m.pair_kind[k] != PAIR_PLANE_CAPSULE) {
      err = "unsupported contact pair kind on the tree (pyramidal) path";
      return false;
    }
    if (m.pair_condim[k] != 3) { err = "pyramidal contacts must have condim 3"; return false; }
    if (D.body_dofmask[b1] != 0u || D.body_dofmask[b2] == 0u) {
      err = "pyramidal contact pairs must be (static geom, moving geom)";
      return false;
    }
    int last = 0;
    for (int d = 0; d < nv; ++d) if ((D.body_dofmask[b2] >> d) & 1u) last = d;
    if (D.dof_ancmask[last] != D.body_dofmask[b2]) { err = "contact body dofs do not form one chain"; return false; }
    for (int s = 0; s < m.pair_ncon[k]; ++s) { D.con_pair[c] = k; D.con_sub[c] = s; D.con_lastdof[c] = last; ++c; }
  }
  if (c != m.ncon) { err = "pair_ncon does not sum to ncon"; return false; }
  if (!D.dense) derive_star(m, D);
  D.nedge = D.dense ? 0 : 4 * m.ncon;
  derive_star_layout(m, D);
  // per-warp slab layout
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
  D.o_xpos = take(3 * nb); D.o_xquat = take(4 * nb); D.o_xmat = take(9 * nb); D.o_xipos = take(3 * nb);
  D.o_cinert = take(CIS * nb); D.o_cdof = take(CDS * nv); D.o_cdofdot = take(CDS * nv);
  D.o_cvel = take(6 * nb); D.o_cacc = take(6 * nb); D.o_cfrc = take(6 * nb);
  // compact-chain M / factor / contact rows and the published solve chains: tree paths only.  The
  // star layout (Ms, Hs, Js, xs) overlays the same block: a launch runs one solver or the other.
  if (!D.dense) {
    const int base = o;
    D.o_Mb = take(nv * DIAL_MAXCHAIN); D.o_L = take(nv * DIAL_MAXCHAIN); D.o_J = take(D.nedge * DIAL_MAXCHAIN);
    D.o_xch = take(nv * DIAL_MAXCHAIN);
    const int generic_end = o;
    o = base;
    if (D.s_on) {
      D.o_Ms = take(D.s_npos * D.s_rs); D.o_Hs = take(D.s_npos * D.s_rs); D.o_Js = take(D.nedge * D.s_rs);
      D.o_xs = take(D.s_npos + 8);
    }
    o = o > generic_end ? o : generic_end;
  } else { D.o_Mb = D.o_L = D.o_J = D.o_xch = 0; }
  D.o_qpos = take(m.nq); D.o_qvel = take(nv); D.o_warm = take(nv); D.o_ctrl = take(m.nu);
  D.o_vec = take(32); D.o_frow = take(32); D.o_cpos = take(3 * m.ncon); D.o_cframe = take(9 * m.ncon);
  D.o_cdist = take(m.ncon); D.o_rcom = take(3 * 4);
  // crb / cfs live from the composite-inertia pass to the mass-matrix rows only, before the solver
  // writes its H rows (star) or M (dense): they overlay that block when it is large enough, which
  // lets 16 warps of the H1 and Allegro models into the 227 KB of shared memory of one CTA.  The
  // star path zeroes the overlaid H rows after use (their padding must read as zero).
  const int ncrb = (CIS + 6) * nb;
  const bool crb_in_Hs = !D.dense && D.s_on && ncrb <= D.s_npos * D.s_rs;
  const bool crb_in_Md = D.dense && ncrb <= nv * nv;
  if (!crb_in_Hs && !crb_in_Md) { D.o_crb = take(CIS * nb); D.o_cfs = take(6 * nb); }
  if (D.dense) {
    // Jd: packed columns (jd_stride); Gd: G rows of one contact at a time (6 x nv); hcs (6x6 cone
    // Hessian) overlays vec|frow (64 contiguous floats, idle while H is assembled).
    // Allegro: 13 KB per warp (crb / cfs in Md) -> 16 warps per CTA.
    D.o_Md = take(nv * nv); D.o_Ld = 0; D.o_Jd = take(D.nrow_c * D.jd_stride); D.o_Gd = take(6 * nv);
    D.o_frow2 = take(D.nrow_c); D.o_cact = take(DIAL_MAXC); D.o_hcs = D.o_vec;
  }
  if (crb_in_Hs) { D.o_crb = D.o_Hs; D.o_cfs = D.o_Hs + CIS * nb; }
  if (crb_in_Md) { D.o_crb = D.o_Md; D.o_cfs = D.o_Md + CIS * nb; }
  D.warp_floats = o;
  return true;
}

// The first field in which `inst` (derived from an instance's model) may not differ from the plan's
// model `plan`, or null.  An instance runs the plan's kernel, launch shape and descriptor, so the integer
// structure must be equal, and so must the floats the plan descriptor copies from the model: timestep
// (n_frames), jnt_range (physical_joint_range) and actuator_ctrlrange (joint_torque_range).
static inline const char* instance_model_difference(const DevModel& plan, const DevModel& inst) {
  const dial_model_desc &a = plan.m, &b = inst.m;
#define DIAL_SAME(f) if (memcmp(&a.f, &b.f, sizeof(a.f)) != 0) return #f;
  DIAL_SAME(nq) DIAL_SAME(nv) DIAL_SAME(nu) DIAL_SAME(nbody) DIAL_SAME(njnt) DIAL_SAME(ngeom) DIAL_SAME(nsite)
  DIAL_SAME(ncon) DIAL_SAME(npair) DIAL_SAME(iterations) DIAL_SAME(ls_iterations) DIAL_SAME(eulerdamp) DIAL_SAME(cone)
  DIAL_SAME(timestep)
  DIAL_SAME(body_parentid) DIAL_SAME(body_rootid) DIAL_SAME(body_depth) DIAL_SAME(body_jntadr) DIAL_SAME(body_dofadr)
  DIAL_SAME(body_dofnum) DIAL_SAME(jnt_type) DIAL_SAME(jnt_qposadr) DIAL_SAME(jnt_dofadr) DIAL_SAME(jnt_limited)
  DIAL_SAME(jnt_range) DIAL_SAME(dof_bodyid) DIAL_SAME(dof_jntid) DIAL_SAME(dof_parentid) DIAL_SAME(geom_type)
  DIAL_SAME(geom_bodyid) DIAL_SAME(pair_kind) DIAL_SAME(pair_geom1) DIAL_SAME(pair_geom2) DIAL_SAME(pair_ncon)
  DIAL_SAME(pair_condim) DIAL_SAME(site_bodyid) DIAL_SAME(actuator_dofadr) DIAL_SAME(actuator_qposadr)
  DIAL_SAME(actuator_ctrllimited) DIAL_SAME(actuator_forcelimited) DIAL_SAME(actuator_ctrlrange)
#undef DIAL_SAME
  // derive_model's tables follow from the fields above, except root_invmass (a float, from body_mass)
  const size_t off = offsetof(DevModel, maxdepth), inv = offsetof(DevModel, root_invmass);
  const char *pa = reinterpret_cast<const char*>(&plan), *pb = reinterpret_cast<const char*>(&inst);
  if (memcmp(pa + off, pb + off, inv - off) != 0 ||
      memcmp(pa + inv + sizeof(plan.root_invmass), pb + inv + sizeof(plan.root_invmass),
             sizeof(DevModel) - inv - sizeof(plan.root_invmass)) != 0)
    return "derived structure";
  return nullptr;
}

// The counts the reward loops over, in range (the kernel indexes the tables with them unchecked).
static inline bool task_valid(const dial_task& t) {
  return t.n_stage >= 1 && t.n_stage <= DIAL_MAXSTAGE && t.n_user >= 0 && t.n_user <= DIAL_MAXUSER;
}

static inline int star_variant(const DevModel& D) {
  if (D.dense) return D.m.nv == DIAL_DENSE_NV ? 3 : -1;   // dense path: one instantiation per library build
  if (D.star_nchain >= 1 && D.star_nchain <= 4) {
    int maxchain = 0;
    for (int i = 0; i < D.m.nv; ++i) maxchain = D.dof_nchain[i] > maxchain ? D.dof_nchain[i] : maxchain;
    if (D.star_nroot == 6 && D.star_maxlen <= 3 && maxchain <= 9) return 1;
    if (D.star_nroot == 7 && D.star_maxlen <= 5) return 2;
    if (D.star_nroot == 6 && D.star_maxlen <= 5) return 4;
  }
  return 0;
}
