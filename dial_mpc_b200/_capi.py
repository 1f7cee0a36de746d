"""ctypes binding of the C ABI in ``include/dial_b200.h``.

The ctypes ``Structure`` classes are generated from the header text itself so the
Python side can never drift from the C layout.  The shared library
``csrc/libdial_b200.so`` is built in-tree by ``__graft_entry__.build()``; importing
this module never falls back to a CPU implementation: a missing library raises.
"""

from __future__ import annotations

import ctypes as C
import os
import re
from typing import Dict, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
HEADER = os.path.join(_ROOT, "include", "dial_b200.h")
LIB_PATH = os.path.join(_HERE, "csrc", "libdial_b200.so")

_CT = {"int32_t": C.c_int32, "uint32_t": C.c_uint32, "float": C.c_float, "int64_t": C.c_int64}


def _parse_header(path: str):
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    defines: Dict[str, int] = {}
    for mm in re.finditer(r"#define\s+(\w+)\s+(\d+)\s*$", text, flags=re.M):
        defines[mm.group(1)] = int(mm.group(2))
    structs = {}
    for mm in re.finditer(r"typedef struct (\w+) \{(.*?)\} (\w+);", text, flags=re.S):
        fields = []
        for stmt in mm.group(2).split(";"):
            stmt = " ".join(stmt.split())
            if not stmt:
                continue
            pm = re.match(r"(const\s+)?(\w+)\s*\*\s*(\w+)$", stmt)
            if pm:  # pointer member
                fields.append((pm.group(3), C.c_void_p))
                continue
            tname, rest = stmt.split(" ", 1)
            base = _CT[tname]
            for decl in rest.split(","):
                decl = decl.strip()
                dm = re.match(r"(\w+)((\[\w+\])*)$", decl)
                name, dims = dm.group(1), re.findall(r"\[(\w+)\]", dm.group(2))
                t = base
                for dname in reversed(dims):
                    t = t * (int(dname) if dname.isdigit() else defines[dname])
                fields.append((name, t))
        structs[mm.group(1)] = fields
    return defines, structs


DEFINES, _STRUCTS = _parse_header(HEADER)


def _mk(name):
    return type(name, (C.Structure,), {"_fields_": _STRUCTS[name]})


dial_model_desc = _mk("dial_model_desc")
dial_plan_desc = _mk("dial_plan_desc")
dial_state = _mk("dial_state")
dial_mpc_buffers = _mk("dial_mpc_buffers")
dial_task = _mk("dial_task")
dial_push = _mk("dial_push")
dial_plant = _mk("dial_plant")
dial_terrain = _mk("dial_terrain")

TASK_FIELDS = tuple(name for name, _ in _STRUCTS["dial_task"])
# the plan descriptor's task block has the layout of dial_task (a plan's own task is read through it)
_T0 = getattr(dial_plan_desc, TASK_FIELDS[0]).offset
if any(getattr(dial_plan_desc, f).offset - _T0 != getattr(dial_task, f).offset for f in TASK_FIELDS):
    raise RuntimeError("include/dial_b200.h: the task block of dial_plan_desc does not have the layout of dial_task")


def task_from_desc(d: dial_plan_desc) -> dial_task:
    """The task fields of a plan descriptor (the reward inputs that differ between tasks), checked."""
    t = dial_task()
    for name in TASK_FIELDS:
        v = getattr(d, name)
        if isinstance(v, C.Array):
            C.memmove(C.addressof(getattr(t, name)), C.addressof(v), C.sizeof(v))
        else:
            setattr(t, name, v)
    return check_task(t)


def task_set_command(t: dial_task, override):
    """Write a randomize_tasks one-step command (``BaseEnv.command_override``: (step, vel[3], ang[3]) or
    None) into ``t`` as ``dial_plan_set_command`` writes it into a plan; returns a key of the values."""
    if override is None:
        t.cmd_step = -1
        _set(t.cmd_vel, np.zeros(3, np.float32))
        _set(t.cmd_ang, np.zeros(3, np.float32))
        return None
    vel, ang = np.float32(override[1]).reshape(3), np.float32(override[2]).reshape(3)
    t.cmd_step = int(override[0])
    _set(t.cmd_vel, vel)
    _set(t.cmd_ang, ang)
    return (int(override[0]), tuple(vel.tolist()), tuple(ang.tolist()))


def task_set_stages(t: dial_task, tables) -> dial_task:
    """Write a jump sequence (pose [n,3], yaw [n], contact_targets [n,4,3], contact_radius [n,4]) into
    ``t`` as ``dial_plan_set_stages`` writes it into a plan (unused rows zeroed)."""
    pose, yaw, tgt, rad = (np.ascontiguousarray(x, dtype=np.float32) for x in tables)
    n = int(pose.shape[0])
    if not 1 <= n <= DEFINES["DIAL_MAXSTAGE"]:
        raise ValueError(f"a jump sequence of {n} stages is out of range (1..{DEFINES['DIAL_MAXSTAGE']})")
    if yaw.shape != (n,) or tgt.shape != (n, 4, 3) or rad.shape != (n, 4):
        raise ValueError("stage tables must have shapes [n,3], [n], [n,4,3], [n,4]")
    t.n_stage = n
    for name, v in (("pose_seq", pose), ("yaw_seq", yaw), ("contact_targets", tgt), ("contact_radius", rad)):
        np.ctypeslib.as_array(getattr(t, name))[...] = 0
        _set(getattr(t, name), v)
    return t


def first_shared_difference(a: dial_plan_desc, b: dial_plan_desc) -> Optional[str]:
    """The first field outside the task (shared by every instance of a plan) in which two plan
    descriptors differ, or None."""
    for name, _ in dial_plan_desc._fields_:
        if name in TASK_FIELDS:
            continue
        va, vb = getattr(a, name), getattr(b, name)
        if isinstance(va, C.Array):
            if bytes(va) != bytes(vb):
                return name
        elif va != vb:
            return name
    return None


def check_task(t: dial_task) -> dial_task:
    """Raise unless the counts the kernels index the tables with are in range (include/dial_b200.h)."""
    if not 1 <= t.n_stage <= DEFINES["DIAL_MAXSTAGE"]:
        raise ValueError(f"dial_task.n_stage = {t.n_stage} is out of range (1..{DEFINES['DIAL_MAXSTAGE']})")
    if not 0 <= t.n_user <= DEFINES["DIAL_MAXUSER"]:
        raise ValueError(f"dial_task.n_user = {t.n_user} is out of range (0..{DEFINES['DIAL_MAXUSER']})")
    return t

ENV_IDS = {"unitree_go2_walk": 0, "unitree_go2_seq_jump": 1, "unitree_h1_walk": 2, "allegro_reorient": 3, "unitree_h1_loco": 4,
           "custom": 5}


def _set(field, value):
    """Copy a numpy array into a (possibly nested) ctypes array field, zero padded."""
    arr = np.ctypeslib.as_array(field)
    value = np.asarray(value)
    if value.size == 0:
        return
    sl = tuple(slice(0, s) for s in value.shape)
    if any(s > d for s, d in zip(value.shape, arr.shape)):
        raise ValueError(f"value of shape {value.shape} exceeds capacity {arr.shape}")
    arr[sl] = value


def fill_model_desc(cm) -> dial_model_desc:
    """CompiledModel (modelc) -> C descriptor."""
    d = dial_model_desc()
    for k in ("nq", "nv", "nu", "nbody", "njnt", "ngeom", "nsite", "npair", "ncon",
              "iterations", "ls_iterations", "cone"):
        setattr(d, k, int(getattr(cm, k)))
    d.eulerdamp = int(bool(cm.eulerdamp))
    for k in ("timestep", "tolerance", "ls_tolerance", "impratio", "meaninertia"):
        setattr(d, k, float(getattr(cm, k)))
    _set(d.gravity, cm.gravity)
    A = cm.arrays
    for k in ("body_parentid", "body_rootid", "body_depth", "body_jntadr", "body_dofadr", "body_dofnum",
              "body_pos", "body_quat", "body_ipos", "body_iquat", "body_mass", "body_inertia",
              "jnt_type", "jnt_qposadr", "jnt_dofadr", "jnt_limited", "jnt_pos", "jnt_axis", "jnt_range",
              "jnt_margin", "jnt_solref", "jnt_solimp",
              "dof_bodyid", "dof_jntid", "dof_parentid", "dof_armature", "dof_damping", "dof_invweight0",
              "qpos0", "geom_type", "geom_bodyid", "geom_pos", "geom_quat", "geom_size",
              "pair_kind", "pair_geom1", "pair_geom2", "pair_ncon", "pair_condim", "pair_friction", "pair_margin",
              "pair_gap", "pair_solref", "pair_solimp", "site_bodyid", "site_pos",
              "actuator_dofadr", "actuator_qposadr", "actuator_ctrllimited", "actuator_forcelimited",
              "actuator_gear", "actuator_gain", "actuator_bias", "actuator_ctrlrange", "actuator_forcerange"):
        _set(getattr(d, k), A[k])
    _set(d.body_invweight0, A["body_invweight0"][:, 0])
    _set(d.body_invweight0_rot, A["body_invweight0"][:, 1])
    return d


def _bind(path: str) -> C.CDLL:
    """dlopen one build of the library and declare its prototypes; checks ABI + struct layout."""
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`."
            " There is no CPU fallback for the DIAL-MPC sampling core.")
    lib = C.CDLL(path)
    lib.dial_abi_version.restype = C.c_int
    lib.dial_last_error.restype = C.c_char_p
    lib.dial_sizeof.restype = C.c_size_t
    lib.dial_sizeof.argtypes = [C.c_int]
    lib.dial_plan_create.restype = C.c_void_p
    lib.dial_plan_create.argtypes = [C.POINTER(dial_model_desc), C.POINTER(dial_plan_desc)]
    lib.dial_plan_destroy.argtypes = [C.c_void_p]
    lib.dial_plan_destroy.restype = None
    P, I, V = C.c_void_p, C.c_int, C.c_void_p
    lib.dial_rollout.argtypes = [V, C.POINTER(dial_state), P, I, I, P, P, P, P, V]
    lib.dial_env_step.argtypes = [V, C.POINTER(dial_state), P, P, P, P, P, P, V]
    lib.dial_env_step_kin.argtypes = [V, C.POINTER(dial_state), P, P, P, P, P, P, P, V]
    lib.dial_plan_set_command.argtypes = [V, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), V]
    F = C.POINTER(C.c_float)
    lib.dial_plan_set_stages.argtypes = [V, C.c_int, F, F, F, F, V]
    lib.dial_pipeline_init.argtypes = [V, P, P, P, P, V]
    U2 = C.POINTER(C.c_uint32)
    lib.dial_reverse_rollout.argtypes = [V, C.POINTER(dial_state), P, U2, P, P, P, V]
    lib.dial_reverse_update.argtypes = [V, P, U2, P, P, P, P, P, V]
    lib.dial_reverse_update_x.argtypes = [V, P, U2, P, P, P, P, P, P, V]
    lib.dial_reverse_update_fused.argtypes = [V, P, P, P, P, P, P, V]
    lib.dial_reverse_trajbar.argtypes = [V, P, I, P, P, P, V]
    lib.dial_exchange_create.argtypes = [V, I, I, P]
    lib.dial_exchange_connect.argtypes = [V, P]
    lib.dial_exchange_status.argtypes = [V, U2]
    lib.dial_reverse_trajectories.argtypes = [V, P, P, P, V]
    lib.dial_key_split.argtypes = [U2, U2, U2]
    lib.dial_key_split.restype = None
    lib.dial_fp32_peak.argtypes = [I, C.POINTER(C.c_float)]
    lib.dial_fp32_peak.restype = C.c_int
    lib.dial_launch_count.argtypes = [V]
    lib.dial_launch_count.restype = C.c_int64
    lib.dial_rollout_wpc.argtypes = [V, I]
    lib.dial_rollout_wpc.restype = C.c_int
    lib.dial_debug_counters.argtypes = [V, C.POINTER(C.c_float)]
    lib.dial_debug_counters.restype = C.c_int
    lib.dial_solver_variant.argtypes = [C.POINTER(dial_model_desc)]
    lib.dial_solver_variant.restype = C.c_int
    lib.dial_custom_reward_id.restype = C.c_char_p
    lib.dial_plan_rollout_kernel.argtypes = [V]
    lib.dial_plan_rollout_kernel.restype = C.c_char_p
    lib.dial_mpc_bind.argtypes = [V, C.POINTER(dial_mpc_buffers), P]
    lib.dial_mpc_bind.restype = C.c_int
    lib.dial_mpc_step.argtypes = [V, I, I, V]
    lib.dial_mpc_step.restype = C.c_int
    lib.dial_plan_get_task.argtypes = [V, C.POINTER(dial_task)]
    lib.dial_plan_get_task.restype = C.c_int
    lib.dial_plan_set_instance_model.argtypes = [V, I, C.POINTER(dial_model_desc), V]
    lib.dial_plan_set_instance_model.restype = C.c_int
    lib.dial_plan_set_ensemble_model.argtypes = [V, I, I, C.POINTER(dial_model_desc), V]
    lib.dial_plan_set_ensemble_model.restype = C.c_int
    lib.dial_plan_set_ensemble_risk.argtypes = [V, I, I, C.c_float, V]
    lib.dial_plan_set_ensemble_risk.restype = C.c_int
    lib.dial_plan_member_rewards.argtypes = [V, P, V]
    lib.dial_plan_member_rewards.restype = C.c_int
    lib.dial_plan_set_ensemble_adapt.argtypes = [V, I, I, C.c_float, C.c_float, C.POINTER(C.c_float), V]
    lib.dial_plan_set_ensemble_adapt.restype = C.c_int
    lib.dial_plan_set_ensemble_belief.argtypes = [V, I, C.POINTER(C.c_float), V]
    lib.dial_plan_set_ensemble_belief.restype = C.c_int
    lib.dial_plan_ensemble_belief.argtypes = [V, P, P, V]
    lib.dial_plan_ensemble_belief.restype = C.c_int
    lib.dial_plan_set_instance_schedule.argtypes = [V, I, C.c_float, I, C.POINTER(C.c_float), V]
    lib.dial_plan_set_instance_schedule.restype = C.c_int
    lib.dial_plan_set_instance_iterations.argtypes = [V, C.POINTER(C.c_int32), V]
    lib.dial_plan_set_instance_iterations.restype = C.c_int
    lib.dial_plan_set_instance_delay.argtypes = [V, I, I, I, V]
    lib.dial_plan_set_instance_delay.restype = C.c_int
    lib.dial_plan_pending_actions.argtypes = [V, P, V]
    lib.dial_plan_pending_actions.restype = C.c_int
    lib.dial_plan_planning_state.argtypes = [V, P, P, P, P, V]
    lib.dial_plan_planning_state.restype = C.c_int
    lib.dial_plan_set_instance_observation.argtypes = [V, I, I, P, P, C.POINTER(C.c_uint32), V]
    lib.dial_plan_set_instance_observation.restype = C.c_int
    lib.dial_plan_observed_state.argtypes = [V, P, P, P, P, P, V]
    lib.dial_plan_observed_state.restype = C.c_int
    lib.dial_plan_set_instance_pushes.argtypes = [V, I, I, C.POINTER(dial_push), V]
    lib.dial_plan_set_instance_pushes.restype = C.c_int
    lib.dial_plan_set_instance_plant.argtypes = [V, I, C.POINTER(dial_plant), V]
    lib.dial_plan_set_instance_plant.restype = C.c_int
    lib.dial_plan_set_instance_terrain.argtypes = [V, I, I, C.POINTER(dial_terrain), V]
    lib.dial_plan_set_instance_terrain.restype = C.c_int
    for fn in ("dial_rollout", "dial_env_step", "dial_env_step_kin", "dial_plan_set_command", "dial_plan_set_stages", "dial_pipeline_init", "dial_reverse_rollout",
               "dial_reverse_update", "dial_reverse_update_x", "dial_reverse_update_fused", "dial_reverse_trajbar",
               "dial_reverse_trajectories", "dial_exchange_create", "dial_exchange_connect", "dial_exchange_status"):
        getattr(lib, fn).restype = C.c_int
    if lib.dial_abi_version() != DEFINES["DIAL_ABI_VERSION"]:
        raise RuntimeError(f"{os.path.basename(path)} ABI version does not match include/dial_b200.h")
    for i, t in enumerate((dial_model_desc, dial_plan_desc, dial_state, dial_mpc_buffers, dial_task, dial_push, dial_plant,
                              dial_terrain)):
        if lib.dial_sizeof(i) != C.sizeof(t):
            raise RuntimeError(f"struct layout mismatch for {t.__name__}: C {lib.dial_sizeof(i)} vs ctypes {C.sizeof(t)}")
    return lib


_LIBS: Dict[str, C.CDLL] = {}


def lib(path: Optional[str] = None) -> C.CDLL:
    """The stock library (default) or a custom-reward build (``dial_mpc_b200.custom``)."""
    # DIAL_B200_LIB: an alternative build of the stock library (kernel experiments, A/B timing)
    path = os.path.abspath(path or os.environ.get("DIAL_B200_LIB") or LIB_PATH)
    if path not in _LIBS:
        _LIBS[path] = _bind(path)
    return _LIBS[path]


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError(f"dial_b200: {lib().dial_last_error().decode()} (rc={rc})")


EXPORTS = ["dial_abi_version", "dial_last_error", "dial_sizeof", "dial_plan_create", "dial_plan_destroy", "dial_rollout",
           "dial_env_step", "dial_env_step_kin", "dial_plan_set_command", "dial_plan_set_stages", "dial_pipeline_init", "dial_reverse_rollout", "dial_reverse_update", "dial_reverse_update_x",
           "dial_reverse_update_fused", "dial_exchange_create", "dial_exchange_connect", "dial_exchange_status",
           "dial_reverse_trajbar", "dial_reverse_trajectories", "dial_key_split", "dial_fp32_peak", "dial_launch_count", "dial_rollout_wpc", "dial_debug_counters",
           "dial_solver_variant", "dial_custom_reward_id", "dial_mpc_bind", "dial_mpc_step", "dial_plan_get_task",
           "dial_plan_rollout_kernel", "dial_plan_set_instance_model", "dial_plan_set_ensemble_model",
           "dial_plan_set_ensemble_risk", "dial_plan_member_rewards", "dial_plan_set_ensemble_adapt",
           "dial_plan_set_ensemble_belief", "dial_plan_ensemble_belief", "dial_plan_set_instance_schedule",
           "dial_plan_set_instance_iterations", "dial_plan_set_instance_delay", "dial_plan_pending_actions",
           "dial_plan_planning_state", "dial_plan_set_instance_observation", "dial_plan_observed_state",
           "dial_plan_set_instance_pushes", "dial_plan_set_instance_plant", "dial_plan_set_instance_terrain"]
