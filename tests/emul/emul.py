"""TEST-ONLY python driver of the CPU warp emulator (tests/emul/emul_main.cpp)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

from dial_mpc_b200 import _capi

_DIR = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.join(_DIR, "..", "..")
_SRCS = [os.path.join(_DIR, "emul_main.cpp"), os.path.join(_DIR, "warp_emul.h"),
         os.path.join(_ROOT, "dial_mpc_b200", "csrc", "dial_device.cuh"),
         os.path.join(_ROOT, "dial_mpc_b200", "csrc", "dial_host.h"),
         os.path.join(_ROOT, "include", "dial_b200.h"), os.path.join(_ROOT, "include", "dial_custom_reward.h")]
# -ffp-contract=off: no operation is fused, so the _rn intrinsic shims round each one as the GPU does (g++ emits
# no FMA on x86-64 without -march in any case)
_FLAGS = ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC"]

_V, _I, _F = C.c_void_p, C.c_int, C.c_float
_MAXRANK = _capi.DEFINES["DIAL_MAXRANK"]


class RolloutArgs(C.Structure):
    """ctypes mirror of RolloutArgs (csrc/dial_device.cuh), checked against the C++ layout at load."""
    _fields_ = ([(f, C.c_int32) for f in ("nrows", "H", "mode", "lockstep", "sync_every", "step0", "stage0",
                                          "rows_per_inst", "us_row", "task_rows")] +
                [(f, _V) for f in ("tasks", "qpos0", "qvel0", "warm0", "us", "eps", "Ybar", "noise")] +
                [("key0", C.c_uint32), ("key1", C.c_uint32)] +
                [(f, _V) for f in ("rewss", "rews", "q", "qd", "xpos", "qpos_out", "qvel_out", "warm_out",
                                   "ctrl_out", "kin_out", "counters_in", "counters_out", "key_dev", "rng_dev",
                                   "row_counter", "dbg")] +
                [("xch_world", C.c_int32), ("xch_rank", C.c_int32), ("xch_mbox", _V * _MAXRANK),
                 ("xch_flags", _V * _MAXRANK), ("xch_seq", _V), ("xch_done", _V), ("models", _V),
                 ("rows_per_model", C.c_int32), ("sched", _V), ("iter_lim", _V), ("iter", C.c_int32),
                 ("terrain", _V)])


# the element type of each array field `launch` takes (tasks: a ctypes array of dial_task; sched: InstSchedule)
_ARRAYS = {**{f: np.float32 for f in ("qpos0", "qvel0", "warm0", "us", "eps", "Ybar", "noise", "rewss", "rews", "q",
                                      "qd", "xpos", "qpos_out", "qvel_out", "warm_out", "ctrl_out", "kin_out")},
           **{f: np.int32 for f in ("counters_in", "counters_out", "iter_lim")},
           **{f: np.uint32 for f in ("key_dev", "rng_dev")}, "tasks": _capi.dial_task, "sched": None}
_SCALARS = ("nrows", "H", "mode", "step0", "stage0", "rows_per_inst", "us_row", "task_rows", "key0", "key1",
            "rows_per_model", "iter")
SIZEOF = dict(DelaySetting=0, ObsSetting=1, ObsRing=2, dial_push=3, PushTable=4, InstSchedule=5)   # emul_sizeof

_EXPORTS = dict(
    emul_rollout_field=([_I, C.POINTER(C.c_size_t)], C.c_char_p), emul_sizeof=([_I], C.c_size_t),
    emul_model_flags=([_V, _V], _I),
    emul_launch=([_V, _V, _I, _V, _V, _I, C.POINTER(RolloutArgs), _I, _I], _I),
    emul_launch_map=([C.POINTER(RolloutArgs), _I, _I, _I, _V, _V], _I),
    emul_cta_instance=([_I] * 6, _I), emul_instance_model_difference=([_V, _V, C.c_char_p, _I], _I),
    emul_risk_derive=([_I, _I, _F, _V, _V], None), emul_risk_reduce=([_V, _I, _I, _I, _F, _V], None),
    emul_adapt_reduce=([_V, _I, _I, _I, _F, _V, _F, _V], None),
    emul_adapt_update=([_V, _V, _V, _I, _I, _F, _V, _V, _V], None),
    emul_delay_queue_step=([_V, _I, _I, _I, _V, _V, _V, _I, _I], _I),
    emul_observe_step=([_V, _V, _V, _I, _I, _I] + [_V] * 22 + [_I], _I),
    emul_push_step=([_V, _V, _I, C.c_double, _V, _V, _V, _V, _I], _I),
    # builds with DIAL_SHAPE_*, DIAL_TERRAIN, DIAL_EMUL_TRACE
    emul_shape_selects=([_V, _V], _I), emul_terrain_height=([_V, _F, _F], _F), emul_trace_take=([_V, _I], _I))

_LIBS = {}


def _check_layout(lib):
    off, i = C.c_size_t(), 0
    names = [f for f, _ in RolloutArgs._fields_]
    while (name := lib.emul_rollout_field(i, C.byref(off))) is not None:
        name = name.decode()
        if i >= len(names) or names[i] != name or getattr(RolloutArgs, name).offset != off.value:
            raise RuntimeError(f"emul: RolloutArgs field {i} ({name}, offset {off.value}) differs from the ctypes mirror")
        i += 1
    if i != len(names) or C.sizeof(RolloutArgs) != off.value:
        raise RuntimeError(f"emul: RolloutArgs has {i} fields and {off.value} bytes, the ctypes mirror "
                           f"{len(names)} and {C.sizeof(RolloutArgs)}")


def build(defines=(), reward_source=None):
    """g++ build of the device code for the lock-step warp emulator (cached per defines and reward file).
    ``defines``: -D values (DIAL_TERRAIN, DIAL_SHAPE_*, DIAL_DENSE_NV=n, ...); ``reward_source``: a custom reward
    file (include/dial_custom_reward.h) compiled in, as dial_mpc_b200.custom does with nvcc."""
    key = (tuple(defines), None if reward_source is None else os.path.abspath(reward_source))
    if key in _LIBS:
        return _LIBS[key]
    cmd = _FLAGS + [f"-D{d}" for d in defines] + ["-I", _DIR]
    if key[1] is not None:
        cmd.append(f'-DDIAL_CUSTOM_REWARD_FILE="{key[1]}"')
    h = hashlib.sha256(" ".join(cmd).encode())
    for s in _SRCS + ([key[1]] if key[1] else []):
        h.update(open(s, "rb").read())
    so = os.path.join(_DIR, f"libdial_emul_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(cmd + ["-o", tmp, _SRCS[0]])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    for name, (args, res) in _EXPORTS.items():
        if hasattr(lib, name):
            f = getattr(lib, name)
            f.argtypes, f.restype = args, res
    _check_layout(lib)
    _LIBS[key] = lib
    return lib


def _model_desc(m):
    return m if isinstance(m, _capi.dial_model_desc) else _capi.fill_model_desc(m)


def _address(lib, name, a):
    """The address of the array `a` of field `name`, after checking its element type and layout."""
    if name not in _ARRAYS:
        raise TypeError(f"emul.launch: {name} is not an array field of RolloutArgs that the emulator takes")
    want = _ARRAYS[name]
    if name == "tasks":
        if not (isinstance(a, C.Array) and a._type_ is want):
            raise TypeError("emul.launch: tasks must be a ctypes array of dial_task")
        return C.addressof(a)
    if not isinstance(a, np.ndarray) or not a.flags.c_contiguous:
        raise TypeError(f"emul.launch: {name} must be a C-contiguous NumPy array")
    if (a.dtype.itemsize != lib.emul_sizeof(SIZEOF["InstSchedule"])) if want is None else a.dtype != want:
        raise TypeError(f"emul.launch: {name} has dtype {a.dtype}")
    return a.ctypes.data


def launch(model_or_env, desc, *, wpc=1, kernel=-1, models=None, terrain=None, defines=(), reward_source=None,
           **fields):
    """One rollout_kernel launch in the emulator, CTA by CTA at ``wpc`` warps per CTA (emul_launch).
    ``model_or_env``: the plan's model (an env: its model and reward; or a dial_model_desc); ``models``: the
    models of the launch's model slots; ``terrain``: dial_terrain entries; ``kernel``: -1 the model's solver
    variant, 0..4 that variant, 5 the shape kernel of a DIAL_SHAPE_* build.  ``fields``: RolloutArgs fields by
    name, scalars or NumPy arrays of the field's element type (None: a null pointer)."""
    if hasattr(model_or_env, "sys"):
        reward_source = reward_source or getattr(model_or_env, "reward_source", None) or None
        model_or_env = model_or_env.sys.model
    lib = build(defines, reward_source)
    A = RolloutArgs()
    for name, v in fields.items():
        if name in _SCALARS:
            setattr(A, name, int(v))
        elif v is not None:
            setattr(A, name, _address(lib, name, v))
    md = _model_desc(model_or_env)
    arr = None if models is None else (_capi.dial_model_desc * len(models))(*map(_model_desc, models))
    ter = None if terrain is None else (_capi.dial_terrain * len(terrain))(*terrain)
    rc = lib.emul_launch(C.byref(md), arr, 0 if models is None else len(models), C.byref(desc), ter,
                         0 if terrain is None else len(terrain), C.byref(A), wpc, kernel)
    if rc != 0:
        raise RuntimeError(f"emul_launch returned {rc}")


def rollout(env, plan_desc, qpos, qvel, warm, step0=0, stage0=0, us=None, eps=None, Ybar=None,
            noise=None, key=(0, 0), mode=0, nrows=None, H=None, want_traj=True, defines=(), kernel=-1):
    m = env.sys
    nq, nv, nu, nb = m.nq, m.nv, m.nu, m.nbody
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
    qpos, qvel, warm, us, eps, Ybar, noise = map(f32, (qpos, qvel, warm, us, eps, Ybar, noise))
    if mode == 0:
        nrows, H = us.shape[0], us.shape[1]
    out = dict(rewss=np.zeros((nrows, H), np.float32), rews=np.zeros(nrows, np.float32),
               q=np.zeros((nrows, H, nq), np.float32), qd=np.zeros((nrows, H, nv), np.float32),
               xpos=np.zeros((nrows, H, nb - 1, 3), np.float32), qpos_out=np.zeros(nq, np.float32),
               qvel_out=np.zeros(nv, np.float32), warm_out=np.zeros(nv, np.float32),
               ctrl_out=np.zeros(nu, np.float32))
    launch(env, plan_desc, kernel=kernel, defines=defines, mode=mode, nrows=nrows, H=H, step0=step0, stage0=stage0,
           qpos0=qpos, qvel0=qvel, warm0=warm, us=us, eps=eps, Ybar=Ybar, noise=noise, key0=key[0], key1=key[1],
           **out)
    return out


class EmulPlan:
    """TEST-ONLY stand-in for dial_mpc_b200.plan.Plan on CPU tensors: stage 1 runs the real
    device code through the warp emulator, stage 2/3 (weights, Ybar, bars) are NumPy.  Used by
    the gloo tests to exercise MBDPI's multi-rank plumbing without a GPU."""

    def __init__(self, env, desc):
        import torch
        self.env, self.desc = env, desc
        self.device = torch.device("cpu")
        m = env.sys
        self.nq, self.nv, self.nu, self.nbody = m.nq, m.nv, m.nu, m.nbody
        self.N, self.Ntotal, self.Hs, self.Hn = desc.Nsample, desc.Ntotal, desc.Hsample, desc.Hnode
        self.launches = 0
        self._traj = None

    def f32(self, x, shape=None):
        import torch
        t = x.to(torch.float32).contiguous() if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, dtype=np.float32))
        if shape is not None:
            assert tuple(t.shape) == tuple(shape)
        return t

    def _np(self, t):
        return None if t is None else t.detach().cpu().numpy()

    def reverse_rollout(self, state, eps, key, Ybar, noise_scale, rews_local):
        ps = state.pipeline_state
        key = (0, 0) if key is None else (int(key[0]), int(key[1]))
        out = rollout(self.env, self.desc, self._np(ps.qpos), self._np(ps.qvel), self._np(ps.qacc_warmstart),
                      step0=int(state.info.get("step", 0)), stage0=int(state.info.get("contact_stage", 0)),
                      eps=self._np(eps), Ybar=self._np(Ybar), noise=self._np(noise_scale), key=key, mode=1,
                      nrows=self.N + 1, H=self.Hs + 1)
        self._traj = out
        rews_local.copy_(self.f32(out["rews"]))
        self.launches += 1

    def _Y0s(self, eps, Ybar, noise):
        Y0s = eps * noise[None, :, None] + Ybar
        Y0s[:, 0] = Ybar[0]
        return np.clip(np.concatenate([Y0s, Ybar[None]], 0), -1, 1)

    def reverse_update(self, eps, key, Ybar, noise_scale, rews_all, Ybar_out, weights=None):
        assert eps is not None, "EmulPlan.reverse_update needs injected eps"
        r = self._np(rews_all).astype(np.float64)
        logp = (r - r[-1]) / r.std() / self.desc.temp_sample
        w = np.exp(logp - logp.max())
        w /= w.sum()
        Y0s = self._Y0s(self._np(eps).astype(np.float64), self._np(Ybar).astype(np.float64), self._np(noise_scale).astype(np.float64))
        Ybar_out.copy_(self.f32(np.einsum("n,nij->ij", w, Y0s)))
        if weights is not None:
            weights.copy_(self.f32(w))

    def reverse_trajbar(self, weights, rank, qbar, qdbar, xbar):
        w = self._np(weights).astype(np.float64)
        off, N = self.desc.shard_offset, self.N
        wl = np.concatenate([w[off:off + N], [w[-1] if rank == 0 else 0.0]])
        t = self._traj
        qbar.copy_(self.f32(np.einsum("n,nij->ij", wl, t["q"]).ravel()))
        qdbar.copy_(self.f32(np.einsum("n,nij->ij", wl, t["qd"]).ravel()))
        xbar.copy_(self.f32(np.einsum("n,nijk->ijk", wl, t["xpos"]).ravel()))
