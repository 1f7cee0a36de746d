"""MJCF-subset model compiler (host side, fp64).

Replaces, for the DIAL-MPC hot path only, what the reference obtains from
``brax.io.mjcf.load(path)`` -> MuJoCo's XML compiler -> ``mjx.put_model``
(reference call sites: dial_mpc/envs/unitree_go2_env.py:95-99,
dial_mpc/envs/unitree_h1_env.py:150-154).  The MuJoCo compiler is a
third-party dependency that is not vendored in the reference tree, so this
module restates the part of its published behaviour the BASELINE models use:

* ``include``, nested ``default`` classes, ``childclass``
* ``compiler angle/autolimits/eulerseq``, ``option`` (+ ``flag eulerdamp``)
* bodies with explicit ``inertial``, ``freejoint``, hinge/slide joints
* plane / sphere / capsule geoms (``fromto`` supported), sites
* ``motor`` / ``position`` actuators on joints, ``contact/exclude``, keyframes
* derived constants at ``qpos0``: ``dof_invweight0``, ``body_invweight0``,
  ``stat.meaninertia`` (MuJoCo ``mj_setConst`` semantics)
* the static list of candidate contact pairs with mixed contact parameters
  (MuJoCo ``mj_contactParam`` semantics, MJX fixed-size contact arrays)

The output is a :class:`CompiledModel` (plain numpy arrays) that can be
serialised to JSON; the JSON blobs for the BASELINE robots are committed under
``dial_mpc_b200/models`` so that nothing needs the reference tree at run time.
"""

from __future__ import annotations

import json
import os
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import numpy as np

# joint types (MuJoCo mjtJoint numbering)
JNT_FREE, JNT_BALL, JNT_SLIDE, JNT_HINGE = 0, 1, 2, 3
# geom types (MuJoCo mjtGeom numbering)
GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE = 0, 1, 2, 3
GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = 4, 5, 6, 7
_GEOM_NAMES = {
    "plane": GEOM_PLANE, "hfield": GEOM_HFIELD, "sphere": GEOM_SPHERE,
    "capsule": GEOM_CAPSULE, "ellipsoid": GEOM_ELLIPSOID,
    "cylinder": GEOM_CYLINDER, "box": GEOM_BOX, "mesh": GEOM_MESH,
}
# contact-pair kinds understood by the oracle and the CUDA kernels
PAIR_PLANE_SPHERE, PAIR_PLANE_CAPSULE = 0, 1
PAIR_SPHERE_SPHERE, PAIR_SPHERE_CAPSULE, PAIR_CAPSULE_CAPSULE = 2, 3, 4

MJ_MINVAL = 1e-15


# --------------------------------------------------------------------------
# small fp64 quaternion helpers (wxyz)
# --------------------------------------------------------------------------
def _qmul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([
        aw * bw - ax * bx - ay * by - az * bz,
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by - ax * bz + ay * bw + az * bx,
        aw * bz + ax * by - ay * bx + az * bw,
    ])


def _qmat(q):
    w, x, y, z = q
    return np.array([
        [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z],
    ])


def _qrot(q, v):
    return _qmat(q) @ np.asarray(v, dtype=np.float64)


def _axisangle_quat(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    s = np.sin(0.5 * angle)
    return np.array([np.cos(0.5 * angle), axis[0] * s, axis[1] * s, axis[2] * s])


def _z2quat(vec):
    """Quaternion rotating +z onto ``vec`` (MuJoCo mjuu_z2quat)."""
    vec = np.asarray(vec, dtype=np.float64)
    n = np.linalg.norm(vec)
    if n < MJ_MINVAL:
        return np.array([1.0, 0.0, 0.0, 0.0])
    vec = vec / n
    z = np.array([0.0, 0.0, 1.0])
    axis = np.cross(z, vec)
    s = np.linalg.norm(axis)
    if s < 1e-10:
        # parallel or anti-parallel
        if vec[2] > 0:
            return np.array([1.0, 0.0, 0.0, 0.0])
        return np.array([0.0, 1.0, 0.0, 0.0])
    axis = axis / s
    ang = np.arctan2(s, vec[2])
    return _axisangle_quat(axis, ang)



# --------------------------------------------------------------------------
# mesh / primitive inertia (bodies without an explicit <inertial>)
# --------------------------------------------------------------------------
def _load_stl(path: str) -> np.ndarray:
    """Binary STL -> triangles [n, 3, 3] (fp64)."""
    import struct
    raw = open(path, "rb").read()
    n = struct.unpack("<I", raw[80:84])[0]
    if len(raw) != 84 + 50 * n:
        raise NotImplementedError(f"{path}: only binary STL meshes are supported")
    rec = np.frombuffer(raw, dtype=np.dtype([("n", "<f4", 3), ("v", "<f4", (3, 3)), ("a", "<u2")]), offset=84, count=n)
    return rec["v"].astype(np.float64)


def _mesh_mass_properties(tri: np.ndarray):
    """Volume, centre of mass and inertia tensor about the COM (unit density) of a closed
    triangle mesh by signed tetrahedra against the origin."""
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    det = np.einsum("ni,ni->n", a, np.cross(b, c))
    vol = det.sum() / 6.0
    sgn = 1.0 if vol >= 0 else -1.0
    det, vol = det * sgn, vol * sgn
    com = (det[:, None] * (a + b + c)).sum(0) / 24.0 / vol
    # second moments  int x_i x_j dV  over the tetrahedra (0,a,b,c)
    S = np.zeros((3, 3))
    for p in (a, b, c):
        S += 2.0 * np.einsum("n,ni,nj->ij", det, p, p)
    for p, q in ((a, b), (a, c), (b, c)):
        S += np.einsum("n,ni,nj->ij", det, p, q) + np.einsum("n,ni,nj->ij", det, q, p)
    S /= 120.0
    I0 = np.trace(S) * np.eye(3) - S                       # inertia about the origin
    I = I0 - vol * (np.dot(com, com) * np.eye(3) - np.outer(com, com))
    return vol, com, I


def _primitive_mass_properties(gtype: int, size: np.ndarray):
    """Volume and inertia (about the centre, unit density) of sphere / capsule / box."""
    if gtype == GEOM_SPHERE:
        r = size[0]
        v = 4.0 / 3.0 * np.pi * r ** 3
        return v, np.eye(3) * (0.4 * v * r * r)
    if gtype == GEOM_CAPSULE:
        r, h = size[0], 2 * size[1]
        vc, vs = np.pi * r * r * h, 4.0 / 3.0 * np.pi * r ** 3
        ixx = vc * (h * h / 12 + r * r / 4) + vs * (0.4 * r * r + 0.375 * r * h + 0.25 * h * h)
        izz = vc * r * r / 2 + vs * 0.4 * r * r
        return vc + vs, np.diag([ixx, ixx, izz])
    if gtype == GEOM_BOX:
        x, y, z = 2 * size
        v = x * y * z
        return v, np.diag([v * (y * y + z * z) / 12, v * (x * x + z * z) / 12, v * (x * x + y * y) / 12])
    raise NotImplementedError(f"geom-derived inertia for geom type {gtype}")


def _floats(s: str) -> np.ndarray:
    return np.array([float(t) for t in s.replace(",", " ").split()], dtype=np.float64)


# --------------------------------------------------------------------------
# XML loading: includes + defaults
# --------------------------------------------------------------------------
def _load_xml(path: str) -> ET.Element:
    root = ET.parse(path).getroot()
    _expand_includes(root, os.path.dirname(os.path.abspath(path)))
    return root


def _expand_includes(elem: ET.Element, base: str) -> None:
    i = 0
    children = list(elem)
    for child in children:
        if child.tag == "include":
            inc = ET.parse(os.path.join(base, child.attrib["file"])).getroot()
            _expand_includes(inc, base)
            idx = list(elem).index(child)
            elem.remove(child)
            for k, sub in enumerate(list(inc)):
                elem.insert(idx + k, sub)
        else:
            _expand_includes(child, base)
        i += 1


_ACT_TAGS = ("motor", "position", "general", "velocity")


class _Defaults:
    """Resolved default classes: class name -> {element tag -> attrib dict}."""

    def __init__(self, root: ET.Element):
        self.classes: Dict[str, Dict[str, Dict[str, str]]] = {"main": {}}
        for d in root.findall("default"):
            self._walk(d, None, top=True)

    def _walk(self, node: ET.Element, parent: Optional[str], top: bool = False) -> None:
        name = node.attrib.get("class", "main" if top else None)
        if name is None:
            raise ValueError("nested <default> without class")
        base = self.classes.get(parent, {}) if parent else self.classes.get("main", {})
        if top and name == "main":
            cur = self.classes["main"]
        else:
            cur = {k: dict(v) for k, v in base.items()}
            self.classes[name] = cur
        for child in node:
            if child.tag == "default":
                continue
            tag = "actuator" if child.tag in _ACT_TAGS else child.tag
            cur.setdefault(tag, {}).update(child.attrib)
        for child in node:
            if child.tag == "default":
                self._walk(child, name)

    def resolve(self, tag: str, elem: ET.Element, childclass: Optional[str]) -> Dict[str, str]:
        cls = elem.attrib.get("class", childclass or "main")
        if cls not in self.classes:
            raise KeyError(f"unknown default class {cls!r}")
        key = "actuator" if tag in _ACT_TAGS else tag
        out = dict(self.classes[cls].get(key, {}))
        out.update(elem.attrib)
        return out


# --------------------------------------------------------------------------
# compiled model
# --------------------------------------------------------------------------
@dataclass
class CompiledModel:
    """Flat, array-only description of one robot + scene (all fp64 / int)."""

    name: str = ""
    # options
    timestep: float = 0.002
    gravity: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, -9.81]))
    iterations: int = 100
    ls_iterations: int = 50
    tolerance: float = 1e-8
    ls_tolerance: float = 0.01
    impratio: float = 1.0
    cone: int = 0  # 0 pyramidal, 1 elliptic
    eulerdamp: bool = True
    meaninertia: float = 1.0
    # sizes
    nq: int = 0
    nv: int = 0
    nu: int = 0
    nbody: int = 0
    njnt: int = 0
    ngeom: int = 0
    nsite: int = 0
    npair: int = 0
    ncon: int = 0
    # arrays are filled by compile(); see compile() for shapes
    arrays: Dict[str, np.ndarray] = field(default_factory=dict)
    names: Dict[str, List[str]] = field(default_factory=dict)
    keyframes: Dict[str, Dict[str, List[float]]] = field(default_factory=dict)

    def __getattr__(self, item):  # convenience: model.body_pos etc.
        arrays = self.__dict__.get("arrays", {})
        if item in arrays:
            return arrays[item]
        raise AttributeError(item)

    # ---- names -----------------------------------------------------------
    def body_id(self, name: str) -> int:
        return self.names["body"].index(name)

    def site_id(self, name: str) -> int:
        return self.names["site"].index(name)

    def geom_id(self, name: str) -> int:
        return self.names["geom"].index(name)

    def keyframe_qpos(self, name: str) -> np.ndarray:
        return np.array(self.keyframes[name]["qpos"], dtype=np.float64)

    # ---- (de)serialisation ----------------------------------------------
    def to_json(self) -> str:
        scal = {k: getattr(self, k) for k in (
            "name", "timestep", "iterations", "ls_iterations", "tolerance",
            "ls_tolerance", "impratio", "cone", "eulerdamp", "meaninertia",
            "nq", "nv", "nu", "nbody", "njnt", "ngeom", "nsite", "npair", "ncon")}
        scal["gravity"] = self.gravity.tolist()
        arr = {k: {"dtype": str(v.dtype), "shape": list(v.shape), "data": v.ravel().tolist()}
               for k, v in self.arrays.items()}
        return json.dumps({"scalars": scal, "arrays": arr, "names": self.names,
                           "keyframes": self.keyframes}, indent=1)

    @staticmethod
    def from_json(text: str) -> "CompiledModel":
        obj = json.loads(text)
        m = CompiledModel()
        for k, v in obj["scalars"].items():
            setattr(m, k, np.array(v, dtype=np.float64) if k == "gravity" else v)
        m.arrays = {k: np.array(v["data"], dtype=np.dtype(v["dtype"])).reshape(v["shape"])
                    for k, v in obj["arrays"].items()}
        m.names = obj["names"]
        m.keyframes = obj["keyframes"]
        return m

    def save(self, path: str) -> None:
        with open(path, "w") as f:
            f.write(self.to_json())

    @staticmethod
    def load(path: str) -> "CompiledModel":
        with open(path) as f:
            return CompiledModel.from_json(f.read())

    def replace_timestep(self, timestep: float) -> "CompiledModel":
        """Mirror of ``sys.tree_replace({"opt.timestep": ...})``
        (reference: dial_mpc/envs/unitree_go2_env.py:98)."""
        import copy
        m = copy.copy(self)
        m.timestep = float(timestep)
        return m

    # float fields ``replace`` accepts, with the name table their entries are named by
    FLOAT_FIELDS = {"body_mass": "body", "body_inertia": "body", "body_ipos": "body", "dof_damping": "joint",
                    "dof_armature": "joint", "actuator_gear": "actuator", "actuator_gain": "actuator",
                    "actuator_bias": "actuator", "pair_friction": "pair", "pair_solref": "pair",
                    "pair_solimp": "pair", "geom_size": "geom"}

    def replace(self, params: Dict[str, Any]) -> "CompiledModel":
        """A copy with float fields replaced, like ``mjx.Model.tree_replace``: ``"opt.timestep"``,
        ``"opt.gravity"`` or a name of ``FLOAT_FIELDS``, each mapped to a full array or to
        ``{name: value}``.  Bodies are named by body name, dofs by joint name (a value per dof of the
        joint, or one for all of them), actuators by actuator name, geoms by geom name and contact pairs
        by the name of the pair's moving geom (geom2).  Derived constants (``body_invweight0``,
        ``dof_invweight0``, ``meaninertia``) are left as they are; ``set_const`` recomputes them."""
        import copy
        m = copy.copy(self)
        m.arrays = dict(self.arrays)
        m.gravity = np.array(self.gravity, dtype=np.float64)
        for key, val in params.items():
            if key == "opt.timestep":
                m.timestep = float(val)
                continue
            if key == "opt.gravity":
                g = np.array(val, dtype=np.float64)
                if g.shape != (3,):
                    raise ValueError(f"opt.gravity needs 3 values, got shape {g.shape}")
                m.gravity = g
                continue
            if key not in self.FLOAT_FIELDS:
                raise KeyError(f"tree_replace: {key!r} is not a replaceable float field (accepted: opt.timestep, "
                               f"opt.gravity, {', '.join(self.FLOAT_FIELDS)}); structure cannot be replaced")
            old = self.arrays[key]
            if not isinstance(val, dict):
                new = np.array(val, dtype=old.dtype)
                if new.shape != old.shape:
                    raise ValueError(f"tree_replace: {key} has shape {old.shape}, got {new.shape}")
                m.arrays[key] = new
                continue
            new = old.copy()
            for name, v in val.items():
                rows = self._entries(self.FLOAT_FIELDS[key], name, key)
                new[rows] = np.broadcast_to(np.asarray(v, dtype=old.dtype), new[rows].shape)
            m.arrays[key] = new
        return m

    def _entries(self, table: str, name: str, key: str):
        """Index (or dof slice) of entry ``name`` of ``table`` in the arrays of field ``key``."""
        if table == "pair":
            geoms = [self.names["geom"][g] for g in self.arrays["pair_geom2"]]
            if name not in geoms:
                raise KeyError(f"tree_replace: {key}: no contact pair whose moving geom is {name!r} (pairs: {geoms})")
            return geoms.index(name)
        if name not in self.names.get(table, []):
            raise KeyError(f"tree_replace: {key}: unknown {table} {name!r} (known: {self.names.get(table, [])})")
        i = self.names[table].index(name)
        if table != "joint":
            return i
        a = self.arrays["jnt_dofadr"][i]
        nd = {0: 6, 1: 3}.get(int(self.arrays["jnt_type"][i]), 1)
        return slice(a, a + nd)

    def set_const(self) -> "CompiledModel":
        """Recompute the constants MuJoCo's ``mj_setConst`` derives at qpos0 (``body_invweight0``,
        ``dof_invweight0``, ``meaninertia``) from the current masses and inertias, in place."""
        _set_const(self)
        return self


# --------------------------------------------------------------------------
# compiler
# --------------------------------------------------------------------------
def _orientation(attr: Dict[str, str], eulerseq: str, degree: bool) -> np.ndarray:
    if "quat" in attr:
        q = _floats(attr["quat"])
        return q / np.linalg.norm(q)
    if "euler" in attr:
        e = _floats(attr["euler"])
        if degree:
            e = np.deg2rad(e)
        q = np.array([1.0, 0.0, 0.0, 0.0])
        for ch, ang in zip(eulerseq, e):
            ax = {"x": [1, 0, 0], "y": [0, 1, 0], "z": [0, 0, 1]}[ch.lower()]
            qi = _axisangle_quat(ax, ang)
            # lower-case: intrinsic (rotating frame) => post-multiply
            q = _qmul(q, qi) if ch.islower() else _qmul(qi, q)
        return q
    if "axisangle" in attr:
        a = _floats(attr["axisangle"])
        ang = np.deg2rad(a[3]) if degree else a[3]
        return _axisangle_quat(a[:3] / np.linalg.norm(a[:3]), ang)
    if "zaxis" in attr:
        return _z2quat(_floats(attr["zaxis"]))
    if "xyaxes" in attr:
        a = _floats(attr["xyaxes"])
        x = a[:3] / np.linalg.norm(a[:3])
        y = a[3:] - x * np.dot(x, a[3:])
        y = y / np.linalg.norm(y)
        z = np.cross(x, y)
        return _mat2quat(np.stack([x, y, z], axis=1))
    return np.array([1.0, 0.0, 0.0, 0.0])


def _mat2quat(R):
    tr = np.trace(R)
    if tr > 0:
        s = np.sqrt(tr + 1.0) * 2
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
        q = np.zeros(4)
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = (R[j, i] + R[i, j]) / s
        q[1 + k] = (R[k, i] + R[i, k]) / s
    return q / np.linalg.norm(q)


def compile_mjcf(path: str, name: Optional[str] = None) -> CompiledModel:
    root = _load_xml(path)
    defaults = _Defaults(root)
    m = CompiledModel(name=name or root.attrib.get("model", os.path.basename(path)))

    # ---- compiler / option ----------------------------------------------
    degree, autolimits, eulerseq = True, True, "xyz"
    meshdir = ""
    for c in root.findall("compiler"):
        if "angle" in c.attrib:
            degree = c.attrib["angle"] == "degree"
        if "autolimits" in c.attrib:
            autolimits = c.attrib["autolimits"] == "true"
        eulerseq = c.attrib.get("eulerseq", eulerseq)
        meshdir = c.attrib.get("meshdir", meshdir)
    for o in root.findall("option"):
        a = o.attrib
        m.timestep = float(a.get("timestep", m.timestep))
        if "gravity" in a:
            m.gravity = _floats(a["gravity"])
        m.iterations = int(a.get("iterations", m.iterations))
        m.ls_iterations = int(a.get("ls_iterations", m.ls_iterations))
        m.tolerance = float(a.get("tolerance", m.tolerance))
        m.ls_tolerance = float(a.get("ls_tolerance", m.ls_tolerance))
        m.impratio = float(a.get("impratio", m.impratio))
        if "cone" in a:
            m.cone = {"pyramidal": 0, "elliptic": 1}[a["cone"]]
        if a.get("solver", "Newton") != "Newton":
            raise NotImplementedError("only the Newton solver is supported")
        if a.get("integrator", "Euler") != "Euler":
            raise NotImplementedError("only the Euler integrator is supported")
        for fl in o.findall("flag"):
            if "eulerdamp" in fl.attrib:
                m.eulerdamp = fl.attrib["eulerdamp"] == "enable"

    # ---- mesh assets (only used for the inertia of bodies without <inertial>) -----------
    mesh_files: Dict[str, str] = {}
    for sec in root.findall("asset"):
        for me in sec.findall("mesh"):
            a = defaults.resolve("mesh", me, None)
            if "file" in a:
                nm = a.get("name", os.path.splitext(os.path.basename(a["file"]))[0])
                mesh_files[nm] = os.path.join(os.path.dirname(os.path.abspath(path)), meshdir, a["file"])
    mesh_cache: Dict[str, Any] = {}

    def mesh_props(name: str):
        if name not in mesh_cache:
            mesh_cache[name] = _mesh_mass_properties(_load_stl(mesh_files[name]))
        return mesh_cache[name]

    # ---- bodies (DFS, document order) ------------------------------------
    bodies: List[Dict[str, Any]] = [dict(name="world", parent=0, pos=np.zeros(3),
                                         quat=np.array([1.0, 0, 0, 0]), ipos=np.zeros(3),
                                         iquat=np.array([1.0, 0, 0, 0]), mass=0.0,
                                         inertia=np.zeros(3), joints=[], depth=0)]
    geoms: List[Dict[str, Any]] = []
    sites: List[Dict[str, Any]] = []

    def add_geom(g: ET.Element, bid: int, childclass: Optional[str]):
        a = defaults.resolve("geom", g, childclass)
        gtype = _GEOM_NAMES[a.get("type", "sphere")]
        contype = int(a.get("contype", 1))
        conaff = int(a.get("conaffinity", 1))
        size = np.zeros(3)
        if "size" in a:
            s = _floats(a["size"])
            size[: len(s)] = s
        pos = _floats(a["pos"]) if "pos" in a else np.zeros(3)
        quat = _orientation(a, eulerseq, degree)
        if "fromto" in a:
            ft = _floats(a["fromto"])
            vec = ft[0:3] - ft[3:6]  # MuJoCo: z-axis points from `to` towards `from`
            pos = 0.5 * (ft[0:3] + ft[3:6])
            quat = _z2quat(vec)
            size[1] = 0.5 * np.linalg.norm(vec)
        fr = np.array([1.0, 0.005, 0.0001])
        if "friction" in a:
            f = _floats(a["friction"])
            fr[: len(f)] = f
        solimp = np.array([0.9, 0.95, 0.001, 0.5, 2.0])
        if "solimp" in a:
            s = _floats(a["solimp"])
            solimp[: len(s)] = s
        solref = np.array([0.02, 1.0])
        if "solref" in a:
            s = _floats(a["solref"])
            solref[: len(s)] = s
        geoms.append(dict(
            mesh=a.get("mesh"), mass_attr=(float(a["mass"]) if "mass" in a else None),
            density=float(a.get("density", 1000.0)),
            name=a.get("name", ""), type=gtype, body=bid, pos=pos, quat=quat, size=size,
            friction=fr, condim=int(a.get("condim", 3)), contype=contype, conaffinity=conaff,
            margin=float(a.get("margin", 0.0)), gap=float(a.get("gap", 0.0)),
            solref=solref, solimp=solimp, solmix=float(a.get("solmix", 1.0)),
            priority=int(a.get("priority", 0))))

    def add_site(s: ET.Element, bid: int, childclass: Optional[str]):
        a = defaults.resolve("site", s, childclass)
        sites.append(dict(name=a.get("name", ""), body=bid,
                          pos=_floats(a["pos"]) if "pos" in a else np.zeros(3),
                          quat=_orientation(a, eulerseq, degree)))

    def walk(elem: ET.Element, parent: int, childclass: Optional[str], depth: int):
        childclass = elem.attrib.get("childclass", childclass)
        b = dict(name=elem.attrib.get("name", ""), parent=parent,
                 pos=_floats(elem.attrib["pos"]) if "pos" in elem.attrib else np.zeros(3),
                 quat=_orientation(elem.attrib, eulerseq, degree), joints=[], depth=depth,
                 ipos=None)
        bid = len(bodies)
        bodies.append(b)
        for ch in elem:
            if ch.tag == "inertial":
                a = ch.attrib
                b["ipos"] = _floats(a["pos"]) if "pos" in a else np.zeros(3)
                b["mass"] = float(a["mass"])
                if "fullinertia" in a:
                    f = _floats(a["fullinertia"])
                    I = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
                    w, V = np.linalg.eigh(I)
                    order = np.argsort(-w)
                    w, V = w[order], V[:, order]
                    if np.linalg.det(V) < 0:
                        V[:, 2] = -V[:, 2]
                    b["inertia"] = w
                    b["iquat"] = _qmul(_orientation(a, eulerseq, degree), _mat2quat(V))
                else:
                    b["inertia"] = _floats(a["diaginertia"])
                    b["iquat"] = _orientation(a, eulerseq, degree)
            elif ch.tag in ("joint", "freejoint"):
                if ch.tag == "freejoint":
                    b["joints"].append(dict(type=JNT_FREE, name=ch.attrib.get("name", ""),
                                            pos=np.zeros(3), axis=np.array([0.0, 0, 1]),
                                            range=np.zeros(2), limited=False, damping=0.0,
                                            armature=0.0, margin=0.0, ref=0.0,
                                            solref=np.array([0.02, 1.0]),
                                            solimp=np.array([0.9, 0.95, 0.001, 0.5, 2.0])))
                    continue
                a = defaults.resolve("joint", ch, childclass)
                jt = {"free": JNT_FREE, "ball": JNT_BALL, "slide": JNT_SLIDE,
                      "hinge": JNT_HINGE}[a.get("type", "hinge")]
                if jt == JNT_BALL:
                    raise NotImplementedError("ball joints are not supported")
                rng = _floats(a["range"]) if "range" in a else np.zeros(2)
                if degree and jt == JNT_HINGE:
                    rng = np.deg2rad(rng)
                if "limited" in a and a["limited"] != "auto":
                    limited = a["limited"] == "true"
                else:
                    limited = autolimits and "range" in a
                axis = _floats(a["axis"]) if "axis" in a else np.array([0.0, 0, 1])
                solimp = np.array([0.9, 0.95, 0.001, 0.5, 2.0])
                if "solimplimit" in a:
                    s = _floats(a["solimplimit"])
                    solimp[: len(s)] = s
                solref = np.array([0.02, 1.0])
                if "solreflimit" in a:
                    s = _floats(a["solreflimit"])
                    solref[: len(s)] = s
                if float(a.get("stiffness", 0.0)) != 0.0 or float(a.get("frictionloss", 0.0)) != 0.0:
                    raise NotImplementedError("joint stiffness / frictionloss not supported")
                b["joints"].append(dict(
                    type=jt, name=a.get("name", ""),
                    pos=_floats(a["pos"]) if "pos" in a else np.zeros(3),
                    axis=axis / np.linalg.norm(axis), range=rng, limited=limited,
                    damping=float(a.get("damping", 0.0)), armature=float(a.get("armature", 0.0)),
                    margin=float(a.get("margin", 0.0)), ref=float(a.get("ref", 0.0)),
                    solref=solref, solimp=solimp))
            elif ch.tag == "geom":
                add_geom(ch, bid, childclass)
            elif ch.tag == "site":
                add_site(ch, bid, childclass)
        if b["ipos"] is None:
            # no explicit inertial: inertia would come from geoms (meshes); the
            # BASELINE Go2/H1 models never need it.  Massless bodies are allowed
            # only when they carry no joint.
            b["ipos"] = np.zeros(3)
            b["iquat"] = np.array([1.0, 0, 0, 0])
            b["mass"] = 0.0
            b["inertia"] = np.zeros(3)
            b["needs_geom_inertia"] = True
        for ch in elem:
            if ch.tag == "body":
                walk(ch, bid, childclass, depth + 1)

    for wb in root.findall("worldbody"):
        cc = wb.attrib.get("childclass")
        for ch in wb:
            if ch.tag == "geom":
                add_geom(ch, 0, cc)
            elif ch.tag == "site":
                add_site(ch, 0, cc)
        for ch in wb:
            if ch.tag == "body":
                walk(ch, 0, cc, 1)

    # geom-derived inertia (MuJoCo inertiafromgeom="auto"): bodies without <inertial>
    for bid, b in enumerate(bodies):
        if bid == 0 or not b.get("needs_geom_inertia"):
            continue
        mass, mcom, parts = 0.0, np.zeros(3), []
        for g in geoms:
            if g["body"] != bid:
                continue
            if g["type"] == GEOM_MESH:
                vol, c_loc, I_loc = mesh_props(g["mesh"])
            elif g["type"] == GEOM_PLANE:
                continue
            else:
                vol, I_loc = _primitive_mass_properties(g["type"], g["size"])
                c_loc = np.zeros(3)
            gm = g["mass_attr"] if g["mass_attr"] is not None else g["density"] * vol
            if gm <= 0.0:
                continue
            scale = gm / vol
            R = _qmat(g["quat"])
            c_b = g["pos"] + R @ c_loc
            parts.append((gm, c_b, R @ (I_loc * scale) @ R.T))
            mass += gm
            mcom += gm * c_b
        if mass <= 0.0:
            if b["joints"]:
                raise NotImplementedError(f"body {b['name']!r} has a joint but neither <inertial> nor massive geoms")
            continue
        mcom /= mass
        I = np.zeros((3, 3))
        for gm, c_b, I_b in parts:
            dvec = c_b - mcom
            I += I_b + gm * (np.dot(dvec, dvec) * np.eye(3) - np.outer(dvec, dvec))
        wv, V = np.linalg.eigh(I)
        order = np.argsort(-wv)
        wv, V = wv[order], V[:, order]
        if np.linalg.det(V) < 0:
            V[:, 2] = -V[:, 2]
        b["mass"], b["ipos"], b["inertia"], b["iquat"] = mass, mcom, wv, _mat2quat(V)

    nbody = len(bodies)
    m.nbody = nbody
    A = m.arrays
    A["body_parentid"] = np.array([b["parent"] for b in bodies], dtype=np.int32)
    A["body_depth"] = np.array([b["depth"] for b in bodies], dtype=np.int32)
    rootid = np.zeros(nbody, dtype=np.int32)
    for i in range(1, nbody):
        p = bodies[i]["parent"]
        rootid[i] = i if p == 0 else rootid[p]
    A["body_rootid"] = rootid
    A["body_pos"] = np.stack([b["pos"] for b in bodies])
    A["body_quat"] = np.stack([b["quat"] for b in bodies])
    A["body_ipos"] = np.stack([b["ipos"] for b in bodies])
    A["body_iquat"] = np.stack([b["iquat"] for b in bodies])
    A["body_mass"] = np.array([b["mass"] for b in bodies], dtype=np.float64)
    A["body_inertia"] = np.stack([b["inertia"] for b in bodies])
    m.names["body"] = [b["name"] for b in bodies]

    # ---- joints / dofs ---------------------------------------------------
    jnt = dict(type=[], bodyid=[], qposadr=[], dofadr=[], pos=[], axis=[], range=[],
               limited=[], margin=[], solref=[], solimp=[])
    dof = dict(bodyid=[], jntid=[], parentid=[], armature=[], damping=[])
    body_jntadr = -np.ones(nbody, dtype=np.int32)
    body_dofadr = -np.ones(nbody, dtype=np.int32)
    body_dofnum = np.zeros(nbody, dtype=np.int32)
    body_lastdof = -np.ones(nbody, dtype=np.int32)  # last dof of the body or its ancestors
    qpos0: List[float] = []
    names_j: List[str] = []
    nq = nv = 0
    for bid, b in enumerate(bodies):
        if len(b["joints"]) > 1:
            raise NotImplementedError("more than one joint per body is not supported")
        last = body_lastdof[b["parent"]] if bid > 0 else -1
        for j in b["joints"]:
            jid = len(jnt["type"])
            body_jntadr[bid] = jid
            body_dofadr[bid] = nv
            names_j.append(j["name"])
            jnt["type"].append(j["type"])
            jnt["bodyid"].append(bid)
            jnt["qposadr"].append(nq)
            jnt["dofadr"].append(nv)
            jnt["pos"].append(j["pos"])
            jnt["axis"].append(j["axis"])
            jnt["range"].append(j["range"])
            jnt["limited"].append(int(j["limited"]))
            jnt["margin"].append(j["margin"])
            jnt["solref"].append(j["solref"])
            jnt["solimp"].append(j["solimp"])
            nd = 6 if j["type"] == JNT_FREE else 1
            body_dofnum[bid] = nd
            for k in range(nd):
                dof["bodyid"].append(bid)
                dof["jntid"].append(jid)
                dof["parentid"].append(last)
                dof["armature"].append(j["armature"])
                dof["damping"].append(j["damping"])
                last = nv
                nv += 1
            if j["type"] == JNT_FREE:
                qpos0.extend(list(b["pos"]) + list(b["quat"]))
                nq += 7
            else:
                qpos0.append(j["ref"])
                nq += 1
        body_lastdof[bid] = last
    m.nq, m.nv, m.njnt = nq, nv, len(jnt["type"])
    A["body_jntadr"], A["body_dofadr"], A["body_dofnum"] = body_jntadr, body_dofadr, body_dofnum
    A["jnt_type"] = np.array(jnt["type"], dtype=np.int32)
    A["jnt_bodyid"] = np.array(jnt["bodyid"], dtype=np.int32)
    A["jnt_qposadr"] = np.array(jnt["qposadr"], dtype=np.int32)
    A["jnt_dofadr"] = np.array(jnt["dofadr"], dtype=np.int32)
    A["jnt_pos"] = np.stack(jnt["pos"])
    A["jnt_axis"] = np.stack(jnt["axis"])
    A["jnt_range"] = np.stack(jnt["range"])
    A["jnt_limited"] = np.array(jnt["limited"], dtype=np.int32)
    A["jnt_margin"] = np.array(jnt["margin"], dtype=np.float64)
    A["jnt_solref"] = np.stack(jnt["solref"])
    A["jnt_solimp"] = np.stack(jnt["solimp"])
    A["dof_bodyid"] = np.array(dof["bodyid"], dtype=np.int32)
    A["dof_jntid"] = np.array(dof["jntid"], dtype=np.int32)
    A["dof_parentid"] = np.array(dof["parentid"], dtype=np.int32)
    A["dof_armature"] = np.array(dof["armature"], dtype=np.float64)
    A["dof_damping"] = np.array(dof["damping"], dtype=np.float64)
    A["qpos0"] = np.array(qpos0, dtype=np.float64)
    m.names["joint"] = names_j

    # ---- geoms (collision-capable only), body-major order ----------------
    col = [g for g in geoms if (g["contype"] | g["conaffinity"]) != 0]
    col.sort(key=lambda g: g["body"])  # stable: keeps document order inside a body
    for g in col:
        if g["type"] not in (GEOM_PLANE, GEOM_SPHERE, GEOM_CAPSULE):
            raise NotImplementedError(f"collision geom type {g['type']} not supported")
    m.ngeom = len(col)
    A["geom_type"] = np.array([g["type"] for g in col], dtype=np.int32)
    A["geom_bodyid"] = np.array([g["body"] for g in col], dtype=np.int32)
    A["geom_pos"] = np.stack([g["pos"] for g in col]) if col else np.zeros((0, 3))
    A["geom_quat"] = np.stack([g["quat"] for g in col]) if col else np.zeros((0, 4))
    A["geom_size"] = np.stack([g["size"] for g in col]) if col else np.zeros((0, 3))
    m.names["geom"] = [g["name"] for g in col]

    # ---- sites -------------------------------------------------------------
    m.nsite = len(sites)
    A["site_bodyid"] = np.array([s["body"] for s in sites], dtype=np.int32)
    A["site_pos"] = np.stack([s["pos"] for s in sites]) if sites else np.zeros((0, 3))
    m.names["site"] = [s["name"] for s in sites]

    # ---- actuators ---------------------------------------------------------
    acts = []
    for sec in root.findall("actuator"):
        for a_el in sec:
            a = defaults.resolve(a_el.tag, a_el, None)
            if "joint" not in a:
                raise NotImplementedError("only joint transmissions are supported")
            jid = names_j.index(a["joint"])
            if A["jnt_type"][jid] == JNT_FREE:
                raise NotImplementedError("actuators on free joints are not supported")
            gear = _floats(a["gear"])[0] if "gear" in a else 1.0
            if a_el.tag == "motor":
                gain, bias = 1.0, np.zeros(3)
            elif a_el.tag == "position":
                kp = float(a.get("kp", 1.0))
                kv = float(a.get("kv", 0.0))
                gain, bias = kp, np.array([0.0, -kp, -kv])
            else:
                raise NotImplementedError(f"actuator <{a_el.tag}> not supported")
            ctrlrange = _floats(a["ctrlrange"]) if "ctrlrange" in a else np.zeros(2)
            forcerange = _floats(a["forcerange"]) if "forcerange" in a else np.zeros(2)
            cl = a.get("ctrllimited", "auto")
            fl = a.get("forcelimited", "auto")
            acts.append(dict(
                name=a.get("name", ""), jnt=jid, gear=gear, gain=gain, bias=bias,
                ctrlrange=ctrlrange, forcerange=forcerange,
                ctrllimited=(cl == "true") or (cl == "auto" and autolimits and "ctrlrange" in a),
                forcelimited=(fl == "true") or (fl == "auto" and autolimits and "forcerange" in a)))
    m.nu = len(acts)
    A["actuator_jntid"] = np.array([a["jnt"] for a in acts], dtype=np.int32)
    A["actuator_dofadr"] = np.array([A["jnt_dofadr"][a["jnt"]] for a in acts], dtype=np.int32)
    A["actuator_qposadr"] = np.array([A["jnt_qposadr"][a["jnt"]] for a in acts], dtype=np.int32)
    A["actuator_gear"] = np.array([a["gear"] for a in acts], dtype=np.float64)
    A["actuator_gain"] = np.array([a["gain"] for a in acts], dtype=np.float64)
    A["actuator_bias"] = np.stack([a["bias"] for a in acts]) if acts else np.zeros((0, 3))
    A["actuator_ctrlrange"] = np.stack([a["ctrlrange"] for a in acts]) if acts else np.zeros((0, 2))
    A["actuator_ctrllimited"] = np.array([int(a["ctrllimited"]) for a in acts], dtype=np.int32)
    A["actuator_forcerange"] = np.stack([a["forcerange"] for a in acts]) if acts else np.zeros((0, 2))
    A["actuator_forcelimited"] = np.array([int(a["forcelimited"]) for a in acts], dtype=np.int32)
    m.names["actuator"] = [a["name"] for a in acts]

    # ---- contact pairs -----------------------------------------------------
    excludes = set()
    for sec in root.findall("contact"):
        for ex in sec.findall("exclude"):
            b1 = m.names["body"].index(ex.attrib["body1"])
            b2 = m.names["body"].index(ex.attrib["body2"])
            excludes.add((min(b1, b2), max(b1, b2)))
        if sec.findall("pair"):
            raise NotImplementedError("explicit contact pairs are not supported")
    weld = np.zeros(nbody, dtype=np.int32)  # body_weldid: nearest ancestor with a joint
    for i in range(1, nbody):
        weld[i] = i if bodies[i]["joints"] else weld[bodies[i]["parent"]]
    pairs = []
    for i1 in range(len(col)):
        for i2 in range(i1 + 1, len(col)):
            g1, g2 = col[i1], col[i2]
            b1, b2 = g1["body"], g2["body"]
            if not ((g1["contype"] & g2["conaffinity"]) or (g2["contype"] & g1["conaffinity"])):
                continue
            if weld[b1] == weld[b2]:
                continue  # same body / both static
            # parent-child filter (MuJoCo filterparent; world parent does not count)
            p1, p2 = weld[bodies[weld[b1]]["parent"]], weld[bodies[weld[b2]]["parent"]]
            if (weld[b1] != 0 and weld[b2] != 0) and (p1 == weld[b2] or p2 == weld[b1]):
                continue
            if (min(b1, b2), max(b1, b2)) in excludes:
                continue
            t1, t2 = g1["type"], g2["type"]
            # MuJoCo orders a pair so that type1 <= type2
            if t1 > t2:
                g1, g2, i1_, i2_ = g2, g1, i2, i1
                t1, t2 = t2, t1
            else:
                i1_, i2_ = i1, i2
            kind = {(GEOM_PLANE, GEOM_SPHERE): PAIR_PLANE_SPHERE,
                    (GEOM_PLANE, GEOM_CAPSULE): PAIR_PLANE_CAPSULE,
                    (GEOM_SPHERE, GEOM_SPHERE): PAIR_SPHERE_SPHERE,
                    (GEOM_SPHERE, GEOM_CAPSULE): PAIR_SPHERE_CAPSULE,
                    (GEOM_CAPSULE, GEOM_CAPSULE): PAIR_CAPSULE_CAPSULE}.get((t1, t2))
            if kind is None:
                raise NotImplementedError(f"collision pair types {(t1, t2)} not supported")
            pairs.append((kind, i1_, i2_, _mix_contact(g1, g2)))
    # MJX concatenates contacts group by group (collision function), then by condim
    order = sorted(range(len(pairs)), key=lambda k: (pairs[k][3]["condim"], pairs[k][0]))
    pairs = [pairs[k] for k in order]
    m.npair = len(pairs)
    ncon_of = {PAIR_PLANE_SPHERE: 1, PAIR_PLANE_CAPSULE: 2, PAIR_SPHERE_SPHERE: 1,
               PAIR_SPHERE_CAPSULE: 1, PAIR_CAPSULE_CAPSULE: 1}
    A["pair_kind"] = np.array([p[0] for p in pairs], dtype=np.int32)
    A["pair_geom1"] = np.array([p[1] for p in pairs], dtype=np.int32)
    A["pair_geom2"] = np.array([p[2] for p in pairs], dtype=np.int32)
    A["pair_ncon"] = np.array([ncon_of[p[0]] for p in pairs], dtype=np.int32)
    A["pair_condim"] = np.array([p[3]["condim"] for p in pairs], dtype=np.int32)
    A["pair_friction"] = np.stack([p[3]["friction"] for p in pairs]) if pairs else np.zeros((0, 5))
    A["pair_margin"] = np.array([p[3]["margin"] for p in pairs], dtype=np.float64)
    A["pair_gap"] = np.array([p[3]["gap"] for p in pairs], dtype=np.float64)
    A["pair_solref"] = np.stack([p[3]["solref"] for p in pairs]) if pairs else np.zeros((0, 2))
    A["pair_solimp"] = np.stack([p[3]["solimp"] for p in pairs]) if pairs else np.zeros((0, 5))
    m.ncon = int(A["pair_ncon"].sum())

    # ---- keyframes ---------------------------------------------------------
    for sec in root.findall("keyframe"):
        for k in sec.findall("key"):
            kf = {}
            for fld in ("qpos", "qvel", "ctrl"):
                if fld in k.attrib:
                    kf[fld] = _floats(k.attrib[fld]).tolist()
            if "qpos" not in kf:
                kf["qpos"] = A["qpos0"].tolist()
            m.keyframes[k.attrib.get("name", f"key{len(m.keyframes)}")] = kf

    _set_const(m)
    return m


def _mix_contact(g1: Dict[str, Any], g2: Dict[str, Any]) -> Dict[str, Any]:
    """MuJoCo ``mj_contactParam`` (as mirrored by MJX's collision driver)."""
    p1, p2 = g1["priority"], g2["priority"]
    if p1 != p2:
        hi = g1 if p1 > p2 else g2
        condim, fr = hi["condim"], hi["friction"].copy()
        mix = 1.0 if p1 > p2 else 0.0
    else:
        condim = max(g1["condim"], g2["condim"])
        fr = np.maximum(g1["friction"], g2["friction"])
        s1, s2 = g1["solmix"], g2["solmix"]
        if s1 >= MJ_MINVAL and s2 >= MJ_MINVAL:
            mix = s1 / (s1 + s2)
        elif s1 < MJ_MINVAL and s2 < MJ_MINVAL:
            mix = 0.5
        elif s1 < MJ_MINVAL:
            mix = 0.0
        else:
            mix = 1.0
    if g1["solref"][0] > 0 and g2["solref"][0] > 0:
        solref = mix * g1["solref"] + (1 - mix) * g2["solref"]
    else:
        solref = np.minimum(g1["solref"], g2["solref"])
    solimp = mix * g1["solimp"] + (1 - mix) * g2["solimp"]
    return dict(condim=condim,
                friction=np.array([fr[0], fr[0], fr[1], fr[2], fr[2]]),
                margin=max(g1["margin"], g2["margin"]), gap=max(g1["gap"], g2["gap"]),
                solref=solref, solimp=solimp)


# --------------------------------------------------------------------------
# constants at qpos0 (MuJoCo mj_setConst): invweights and mean inertia
# --------------------------------------------------------------------------
def kinematics_fp64(m: CompiledModel, qpos: np.ndarray):
    """Forward kinematics for one configuration (fp64, unbatched)."""
    A = m.arrays
    nb = m.nbody
    xpos = np.zeros((nb, 3))
    xquat = np.zeros((nb, 4))
    xquat[0, 0] = 1.0
    anchor = np.zeros((nb, 3))
    axis = np.zeros((nb, 3))
    for b in range(1, nb):
        p = A["body_parentid"][b]
        pos = xpos[p] + _qrot(xquat[p], A["body_pos"][b])
        quat = _qmul(xquat[p], A["body_quat"][b])
        j = A["body_jntadr"][b]
        if j >= 0:
            qa = A["jnt_qposadr"][j]
            jt = A["jnt_type"][j]
            if jt == JNT_FREE:
                pos = qpos[qa:qa + 3].copy()
                quat = qpos[qa + 3:qa + 7] / np.linalg.norm(qpos[qa + 3:qa + 7])
                anchor[b] = pos
                axis[b] = [0, 0, 1]
            else:
                anchor[b] = pos + _qrot(quat, A["jnt_pos"][j])
                axis[b] = _qrot(quat, A["jnt_axis"][j])
                if jt == JNT_HINGE:
                    quat = _qmul(quat, _axisangle_quat(A["jnt_axis"][j], qpos[qa] - A["qpos0"][qa]))
                    pos = anchor[b] - _qrot(quat, A["jnt_pos"][j])
                else:
                    pos = pos + axis[b] * (qpos[qa] - A["qpos0"][qa])
        xpos[b], xquat[b] = pos, quat / np.linalg.norm(quat)
    xipos = np.stack([xpos[b] + _qrot(xquat[b], A["body_ipos"][b]) for b in range(nb)])
    ximat = np.stack([_qmat(_qmul(xquat[b], A["body_iquat"][b])) for b in range(nb)])
    return xpos, xquat, xipos, ximat, anchor, axis


def body_jacobian_fp64(m: CompiledModel, kin, body: int, point: np.ndarray):
    """Translational / rotational Jacobians (3 x nv) of ``point`` fixed to ``body``."""
    A = m.arrays
    xpos, xquat, _, _, anchor, axis = kin
    jp, jr = np.zeros((3, m.nv)), np.zeros((3, m.nv))
    b = body
    while b > 0:
        j = A["body_jntadr"][b]
        if j >= 0:
            d = A["jnt_dofadr"][j]
            jt = A["jnt_type"][j]
            if jt == JNT_FREE:
                R = _qmat(xquat[b])
                for i in range(3):
                    jp[i, d + i] = 1.0
                    jr[:, d + 3 + i] = R[:, i]
                    jp[:, d + 3 + i] = np.cross(R[:, i], point - xpos[b])
            elif jt == JNT_HINGE:
                jr[:, d] = axis[b]
                jp[:, d] = np.cross(axis[b], point - anchor[b])
            else:
                jp[:, d] = axis[b]
        b = A["body_parentid"][b]
    return jp, jr


def mass_matrix_fp64(m: CompiledModel, qpos: np.ndarray) -> np.ndarray:
    """Joint-space inertia via summed body Jacobians (independent of the CRB code
    paths of the oracle and the CUDA kernels; also used by the tests)."""
    A = m.arrays
    kin = kinematics_fp64(m, qpos)
    _, _, xipos, ximat, _, _ = kin
    M = np.diag(A["dof_armature"].astype(np.float64))
    for b in range(1, m.nbody):
        if A["body_mass"][b] == 0.0:
            continue
        jp, jr = body_jacobian_fp64(m, kin, b, xipos[b])
        Iw = ximat[b] @ np.diag(A["body_inertia"][b]) @ ximat[b].T
        M += A["body_mass"][b] * jp.T @ jp + jr.T @ Iw @ jr
    return M


def _set_const(m: CompiledModel) -> None:
    A = m.arrays
    if m.nv == 0:
        A["dof_invweight0"] = np.zeros(0)
        A["body_invweight0"] = np.zeros((m.nbody, 2))
        return
    q0 = A["qpos0"]
    M = mass_matrix_fp64(m, q0)
    Minv = np.linalg.inv(M)
    m.meaninertia = float(np.mean(np.diag(M)))
    kin = kinematics_fp64(m, q0)
    biw = np.zeros((m.nbody, 2))
    for b in range(1, m.nbody):
        if A["body_dofadr"][b] < 0 and A["body_parentid"][b] == 0:
            # static body welded to the world
            has_dof = False
            bb = b
            while bb > 0:
                if A["body_jntadr"][bb] >= 0:
                    has_dof = True
                bb = A["body_parentid"][bb]
            if not has_dof:
                continue
        jp, jr = body_jacobian_fp64(m, kin, b, kin[2][b])
        biw[b, 0] = np.trace(jp @ Minv @ jp.T) / 3.0
        biw[b, 1] = np.trace(jr @ Minv @ jr.T) / 3.0
    A["body_invweight0"] = biw
    diw = np.diag(Minv).copy()
    for j in range(m.njnt):
        if A["jnt_type"][j] == JNT_FREE:
            d = A["jnt_dofadr"][j]
            diw[d:d + 3] = diw[d:d + 3].mean()
            diw[d + 3:d + 6] = diw[d + 3:d + 6].mean()
    A["dof_invweight0"] = diw
