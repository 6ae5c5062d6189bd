"""The refusal codes of the C entry points that have a 16-bit twin, pinned case by case.

Each fp32 entry point in `PAIRS` and its `_v16` twin start from a well-formed argument set (pointers into one 256-byte
aligned host buffer, small valid sizes, vol_type = B200DRR_VOL_F16).  Every case changes one argument to an invalid value,
or combines one change that is refused with B200DRR_EUNSUPPORTED with one refused with B200DRR_EINVAL, so the order of
those two checks is pinned too.  `EXPECTED` holds the code each case returned when the table was recorded; a case the
library accepted is not in it, so no call here is ever meant to reach CUDA.

The calls run in a child process that sees no CUDA device: a call the library wrongly accepts fails there with a CUDA
error instead of launching a kernel on host pointers.  Without a device the brick kernels' tensor-map encoder is also
missing, so the brick entry points refuse whatever passes their first B200DRR_EINVAL checks with B200DRR_EUNSUPPORTED.

`python tests/test_abi_refusals.py` prints the table for the library `B200DRR_LIB` (default: the in-tree build) names.
"""
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from diffdrr_b200 import _lib  # noqa: E402

EINVAL, EUNSUPPORTED, VOL_F16 = -1, -2, 1

_RAYS = "src tgt raylen out"
_FLAT = "B N voxel_shift eps"
_GRID = "B H W voxel_shift eps"
_POSE = "src G Wd rows cols"
_TRI = "n_points alpha_range"
_MOTION_RAYS = "src tgt raylen"
_MOTION_TAIL = "voxel_shift eps n_points alpha_range stream"
# the fp32 entry point's parameters; its twin takes vol_type after `vol` (after `vol packed` for polyrigid and deform)
PAIRS = {
    "siddon_fwd": f"vol D0 D1 D2 {_RAYS} {_FLAT} reduce align_corners stream",
    "siddon_fwd_sens": f"vol D0 D1 D2 {_RAYS} sens {_FLAT} stream",
    "siddon_fwd_sorted": f"vol D0 D1 D2 {_RAYS} {_FLAT} stream",
    "siddon_fwd_sens_sorted": f"vol D0 D1 D2 {_RAYS} sens {_FLAT} stream",
    "siddon_fwd_grid": f"vol D0 D1 D2 {_RAYS} {_GRID} variant stream",
    "siddon_fwd_sens_grid": f"vol D0 D1 D2 {_RAYS} sens {_GRID} variant stream",
    "siddon_fwd_brick": f"vol D0 D1 D2 src tgt raylen G Wd rows cols out workspace workspace_bytes {_GRID} variant stream",
    "siddon_fwd_brick_subset": "vol D0 D1 D2 src tgt raylen pix_index corners out workspace workspace_bytes B H W Nsub "
                               "voxel_shift eps variant stream",
    "siddon_fwd_pose": f"vol D0 D1 D2 {_POSE} out {_GRID} stream",
    "siddon_fwd_sens_pose": f"vol D0 D1 D2 {_POSE} out sens {_GRID} stream",
    "siddon_fwd_sens_structures": f"vol labels D0 D1 D2 {_POSE} slot_of_label box out sens B S H W voxel_shift eps stream",
    "pack_corners": "vol D0 D1 D2 packed stream",
    "trilinear_fwd": f"vol D0 D1 D2 {_RAYS} {_FLAT} {_TRI} reduce align_corners stream",
    "trilinear_fwd_grid": f"vol D0 D1 D2 {_RAYS} {_GRID} {_TRI} variant stream",
    "trilinear_fwd_sens": f"vol D0 D1 D2 {_RAYS} sens B N H W voxel_shift eps {_TRI} align_corners stream",
    "trilinear_fwd_packed": f"packed D0 D1 D2 {_RAYS} {_GRID} {_TRI} slab stream",
    "trilinear_fwd_sens_packed": f"packed D0 D1 D2 {_RAYS} sens {_GRID} {_TRI} slab stream",
    "trilinear_fwd_sens_pose": f"packed D0 D1 D2 {_POSE} out sens {_GRID} {_TRI} slab stream",
    "polyrigid_fwd": f"vol packed D0 D1 D2 {_MOTION_RAYS} M Bm K weights g0 g1 g2 out B N H W {_MOTION_TAIL}",
    "polyrigid_bwd": f"vol packed D0 D1 D2 {_MOTION_RAYS} M Bm K weights g0 g1 g2 gout g_src g_tgt g_raylen g_M g_alpha_range "
                     f"scratch B N H W {_MOTION_TAIL}",
    "polyrigid_jac": f"vol packed D0 D1 D2 {_MOTION_RAYS} M Bm K weights g0 g1 g2 T img J rects B H W {_MOTION_TAIL}",
    "deform_fwd": f"vol packed D0 D1 D2 {_MOTION_RAYS} field Bf g0 g1 g2 out B N H W {_MOTION_TAIL}",
    "deform_bwd": f"vol packed D0 D1 D2 {_MOTION_RAYS} field Bf g0 g1 g2 gout g_src g_tgt g_raylen g_field g_alpha_range "
                  f"scratch B N H W {_MOTION_TAIL}",
    "deform_jvp": f"vol packed D0 D1 D2 {_MOTION_RAYS} field Bf g0 g1 g2 tangent img jv B N H W {_MOTION_TAIL}",
}

# well-formed values; every other parameter is a pointer into the buffer
GOOD = dict(D0=4, D1=4, D2=8, B=2, H=2, W=2, N=4, Nsub=3, S=2, K=2, Bm=1, Bf=1, g0=2, g1=2, g2=2, n_points=4, reduce=0,
            align_corners=0, variant=0, slab=0, voxel_shift=0.5, eps=1e-8, vol_type=VOL_F16, stream=None,
            workspace_bytes=None)  # the brick workspace size is the library's own answer (see _args)
# one bad value per case
BAD = dict(D0=(0, -1), D1=(0, -1), D2=(0, -1, 6), g0=(0, -1), g1=(0, -1), g2=(0, -1), H=(0, -1, 1), W=(0, -1, 1),
           B=(0, -1, 65536), N=(0, -1, 5), Nsub=(0, 5), S=(0, 257), K=(0, 9), Bm=(0, 3), Bf=(0, 3), n_points=(1,),
           reduce=(1, 2, -1), align_corners=(1,), variant=(1,), slab=(-1,), vol_type=(0, 3))
# changes of several arguments at once, one refusal each
GROUPS = {
    "too_big": dict(D0=2048, D1=1024, D2=1024),
    "lattice_too_big": dict(g0=1024, g1=1024, g2=512),
}
# the changes paired with each other, besides a NULL first pointer: one refused with EUNSUPPORTED, one with EINVAL
COMPETING = {
    EUNSUPPORTED: ("too_big", "lattice_too_big", "K:9", "variant:1", "D2:6", "H:1", "vol:+4"),
    EINVAL: ("B:65536", "vol_type:0", "workspace_bytes:short", "workspace:+4", "packed:only+4", "packed:+4", "weights:+4",
             "field:+4", "g_field:+4", "tangent:+4", "Bm:3", "Bf:3", "n_points:1"),
}
BUF_SLOTS, SLOT = 64, 256


def _params(name, twin):
    p = PAIRS[name].split()
    if twin:
        p.insert(2 if name.startswith(("polyrigid", "deform")) else 1, "vol_type")
    return p


def _optional(name, param):
    # polyrigid / deform take exactly one of vol and packed; the brick entry points walk tgt/raylen rays when G is NULL
    return param == "stream" or (param == "packed" and name.startswith(("polyrigid", "deform"))) or (
        param in ("G", "Wd", "rows", "cols") and name.startswith("siddon_fwd_brick"))


def _mutations(name, twin):
    """label -> {parameter: value}; a pointer value is a slot index into the buffer, or ("+4", slot), or None."""
    params = _params(name, twin)
    ptrs = [q for q in params if q not in GOOD and not _optional(name, q)]
    muts = {}
    for q in ptrs:
        muts[f"{q}:null"] = {q: None}
        muts[f"{q}:+4"] = {q: ("+4", params.index(q))}
    for q, values in BAD.items():
        if q in params:
            for v in values:
                muts[f"{q}:{v}"] = {q: v}
    if "workspace_bytes" in params:
        muts["workspace_bytes:short"] = {"workspace_bytes": "short"}
        muts["workspace_bytes:0"] = {"workspace_bytes": 0}
    if "G" in params and _optional(name, "G"):
        muts["G:set"] = {"G": params.index("G")}
    if "packed" in params and _optional(name, "packed"):
        muts["packed:set"] = {"packed": params.index("packed")}
        muts["packed:only+4"] = {"vol": None, "packed": ("+4", params.index("packed"))}
    muts["too_big"] = dict(GROUPS["too_big"])
    if "g0" in params:
        muts["lattice_too_big"] = dict(GROUPS["lattice_too_big"])
    return muts


def _args(lib, name, twin, change, base):
    params = _params(name, twin)
    vals = {q: GOOD.get(q, params.index(q)) for q in params}
    for q in params:
        if _optional(name, q):
            vals[q] = None
    if "workspace_bytes" in params:
        h, w = (1, GOOD["Nsub"]) if name.endswith("subset") else (GOOD["H"], GOOD["W"])
        vals["workspace_bytes"] = lib.b200drr_siddon_brick_workspace_bytes(GOOD["B"], h, w)
    for q, v in change.items():
        vals[q] = vals["workspace_bytes"] - 1 if v == "short" else v
    out = []
    for q in params:
        v = vals[q]
        if q not in GOOD and v is not None:  # pointer
            v = base + SLOT * v[1] + 4 if isinstance(v, tuple) else base + SLOT * v
        out.append(v)
    return out


def _entry(name, twin):
    return f"b200drr_{name}_v16" if twin else f"b200drr_{name}"


def _run(lib_path, todo):
    """{entry: [label]} -> {entry: {label: code}}, called in a process that sees no CUDA device."""
    lib = ctypes.CDLL(lib_path)
    for fn, (restype, argtypes) in _lib._SIGNATURES.items():
        getattr(lib, fn).restype, getattr(lib, fn).argtypes = restype, argtypes
    raw = ctypes.create_string_buffer(BUF_SLOTS * SLOT + 256)
    base = (ctypes.addressof(raw) + 255) // 256 * 256
    got = {}
    for entry, labels in todo.items():
        twin = entry.endswith("_v16")
        name = entry[len("b200drr_"):-4] if twin else entry[len("b200drr_"):]
        muts = _mutations(name, twin)
        fn = getattr(lib, entry)
        assert len(_params(name, twin)) == len(fn.argtypes), entry
        got[entry] = {}
        for label in labels:
            change = {}
            for part in label.split("&"):
                change.update(muts[part])
            assert change, "a well-formed call is never made"
            got[entry][label] = fn(*_args(lib, name, twin, change, base))
    return got


def _in_child(todo):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    code = f"import json, sys; sys.path.insert(0, {os.path.dirname(__file__)!r}); import test_abi_refusals as t; " \
           f"print(json.dumps(t._run({_lib.lib_path()!r}, json.load(sys.stdin))))"
    proc = subprocess.run([sys.executable, "-c", code], input=json.dumps(todo), capture_output=True, text=True, env=env,
                          timeout=600)
    assert proc.returncode == 0, proc.stderr
    return json.loads(proc.stdout.strip().splitlines()[-1])


def _record():
    """Every single change, then pairs of an EUNSUPPORTED and an EINVAL change among `COMPETING`; keeps the refused cases."""
    entries = {_entry(n, t): (n, t) for n in PAIRS for t in (False, True)}
    single = _in_child({e: list(_mutations(*nt)) for e, nt in entries.items()})
    pairs = {}
    for e, codes in single.items():
        first_ptr = _params(*entries[e])[0] + ":null"
        unsup = [label for label in COMPETING[EUNSUPPORTED] if codes.get(label) == EUNSUPPORTED]
        inval = [label for label in (first_ptr, *COMPETING[EINVAL]) if codes.get(label) == EINVAL]
        pairs[e] = [f"{u}&{i}" for u in unsup for i in inval if set(_mutations(*entries[e])[u]).isdisjoint(
            _mutations(*entries[e])[i])]
    both = _in_child(pairs)
    return {e: {label: c for label, c in {**single[e], **both[e]}.items() if c < 0} for e in entries}


# recorded with `python tests/test_abi_refusals.py`
EXPECTED = {
    'b200drr_siddon_fwd': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1,
        'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'reduce:2': -1,
        'reduce:-1': -1,
    },
    'b200drr_siddon_fwd_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1,
        'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'reduce:1': -1,
        'reduce:2': -1, 'reduce:-1': -1, 'align_corners:1': -1, 'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_siddon_fwd_sens': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1,
        'N:-1': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_sens_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1,
        'N:-1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
        'too_big&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_sorted': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1,
        'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'too_big': -2,
        'too_big&vol:null': -1, 'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_sorted_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1,
        'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'vol_type:0': -1,
        'vol_type:3': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_sens_sorted': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1,
        'N:-1': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_sens_sorted_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1,
        'N:-1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
        'too_big&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_grid': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1,
        'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1,
        'B:65536': -1,
    },
    'b200drr_siddon_fwd_grid_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1,
        'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1,
        'B:65536': -1, 'variant:1': -2, 'vol_type:0': -1, 'vol_type:3': -1, 'variant:1&vol:null': -1, 'variant:1&B:65536': -1,
        'variant:1&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_sens_grid': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1,
        'B:-1': -1, 'B:65536': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_sens_grid_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1,
        'B:-1': -1, 'B:65536': -1, 'variant:1': -2, 'vol_type:0': -1, 'vol_type:3': -1, 'too_big': -2, 'too_big&vol:null': -1,
        'too_big&B:65536': -1, 'too_big&vol_type:0': -1, 'variant:1&vol:null': -1, 'variant:1&B:65536': -1,
        'variant:1&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_brick': {
        'vol:null': -1, 'vol:+4': -2, 'src:null': -1, 'src:+4': -2, 'tgt:null': -1, 'tgt:+4': -2, 'raylen:null': -1,
        'raylen:+4': -2, 'out:null': -1, 'out:+4': -2, 'workspace:null': -1, 'workspace:+4': -2, 'D0:0': -1, 'D0:-1': -1,
        'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'D2:6': -2, 'H:0': -1, 'H:-1': -1, 'H:1': -2, 'W:0': -1, 'W:-1': -1,
        'W:1': -2, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'variant:1': -2, 'workspace_bytes:short': -2, 'workspace_bytes:0': -2,
        'G:set': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'variant:1&vol:null': -1,
        'variant:1&B:65536': -1, 'D2:6&vol:null': -1, 'D2:6&B:65536': -1, 'H:1&vol:null': -1, 'H:1&B:65536': -1,
        'vol:+4&B:65536': -1,
    },
    'b200drr_siddon_fwd_brick_v16': {
        'vol:null': -1, 'vol:+4': -2, 'src:null': -1, 'src:+4': -2, 'tgt:null': -1, 'tgt:+4': -2, 'raylen:null': -1,
        'raylen:+4': -2, 'out:null': -1, 'out:+4': -2, 'workspace:null': -1, 'workspace:+4': -2, 'D0:0': -1, 'D0:-1': -1,
        'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'D2:6': -2, 'H:0': -1, 'H:-1': -1, 'H:1': -2, 'W:0': -1, 'W:-1': -1,
        'W:1': -2, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'variant:1': -2, 'vol_type:0': -1, 'vol_type:3': -1,
        'workspace_bytes:short': -2, 'workspace_bytes:0': -2, 'G:set': -1, 'too_big': -2, 'too_big&vol:null': -1,
        'too_big&B:65536': -1, 'too_big&vol_type:0': -1, 'variant:1&vol:null': -1, 'variant:1&B:65536': -1,
        'variant:1&vol_type:0': -1, 'D2:6&vol:null': -1, 'D2:6&B:65536': -1, 'D2:6&vol_type:0': -1, 'H:1&vol:null': -1,
        'H:1&B:65536': -1, 'H:1&vol_type:0': -1, 'vol:+4&B:65536': -1, 'vol:+4&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_brick_subset': {
        'vol:null': -1, 'vol:+4': -2, 'src:null': -1, 'src:+4': -2, 'tgt:null': -1, 'tgt:+4': -2, 'raylen:null': -1,
        'raylen:+4': -2, 'pix_index:null': -1, 'pix_index:+4': -2, 'corners:null': -1, 'corners:+4': -2, 'out:null': -1,
        'out:+4': -2, 'workspace:null': -1, 'workspace:+4': -2, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'D2:6': -2, 'H:0': -1, 'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1,
        'B:65536': -1, 'Nsub:0': -1, 'Nsub:5': -1, 'variant:1': -2, 'workspace_bytes:short': -2, 'workspace_bytes:0': -2,
        'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'variant:1&vol:null': -1, 'variant:1&B:65536': -1,
        'D2:6&vol:null': -1, 'D2:6&B:65536': -1, 'vol:+4&B:65536': -1,
    },
    'b200drr_siddon_fwd_brick_subset_v16': {
        'vol:null': -1, 'vol:+4': -2, 'src:null': -1, 'src:+4': -2, 'tgt:null': -1, 'tgt:+4': -2, 'raylen:null': -1,
        'raylen:+4': -2, 'pix_index:null': -1, 'pix_index:+4': -2, 'corners:null': -1, 'corners:+4': -2, 'out:null': -1,
        'out:+4': -2, 'workspace:null': -1, 'workspace:+4': -2, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'D2:6': -2, 'H:0': -1, 'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1,
        'B:65536': -1, 'Nsub:0': -1, 'Nsub:5': -1, 'variant:1': -2, 'vol_type:0': -1, 'vol_type:3': -1,
        'workspace_bytes:short': -2, 'workspace_bytes:0': -2, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
        'too_big&vol_type:0': -1, 'variant:1&vol:null': -1, 'variant:1&B:65536': -1, 'variant:1&vol_type:0': -1,
        'D2:6&vol:null': -1, 'D2:6&B:65536': -1, 'D2:6&vol_type:0': -1, 'vol:+4&B:65536': -1, 'vol:+4&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_pose': {
        'vol:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1, 'out:null': -1,
        'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1,
        'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_pose_v16': {
        'vol:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1, 'out:null': -1,
        'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1,
        'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'too_big': -2, 'too_big&vol:null': -1,
        'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_sens_pose': {
        'vol:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1, 'out:null': -1,
        'sens:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1,
        'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'too_big': -2, 'too_big&vol:null': -1,
        'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_sens_pose_v16': {
        'vol:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1, 'out:null': -1,
        'sens:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1,
        'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'too_big': -2,
        'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
    },
    'b200drr_siddon_fwd_sens_structures': {
        'vol:null': -1, 'labels:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1,
        'slot_of_label:null': -1, 'box:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'S:0': -1, 'S:257': -1,
        'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
    },
    'b200drr_siddon_fwd_sens_structures_v16': {
        'vol:null': -1, 'labels:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1,
        'slot_of_label:null': -1, 'box:null': -1, 'out:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'S:0': -1, 'S:257': -1,
        'vol_type:0': -1, 'vol_type:3': -1, 'too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
        'too_big&vol_type:0': -1,
    },
    'b200drr_pack_corners': {
        'vol:null': -1, 'packed:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1,
    },
    'b200drr_pack_corners_v16': {
        'vol:null': -1, 'packed:null': -1, 'packed:+4': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_trilinear_fwd': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'alpha_range:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1,
        'N:-1': -1, 'n_points:1': -1, 'reduce:2': -1, 'reduce:-1': -1,
    },
    'b200drr_trilinear_fwd_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'alpha_range:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1,
        'N:-1': -1, 'n_points:1': -1, 'reduce:1': -1, 'reduce:2': -1, 'reduce:-1': -1, 'align_corners:1': -1, 'vol_type:0': -1,
        'vol_type:3': -1,
    },
    'b200drr_trilinear_fwd_grid': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'alpha_range:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1,
        'B:-1': -1, 'B:65536': -1, 'n_points:1': -1,
    },
    'b200drr_trilinear_fwd_grid_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'alpha_range:null': -1, 'D0:0': -1,
        'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1,
        'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_trilinear_fwd_sens': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1,
        'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:-1': -1,
        'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1,
        'n_points:1': -1, 'align_corners:1': -1,
    },
    'b200drr_trilinear_fwd_sens_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1,
        'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:-1': -1,
        'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1,
        'n_points:1': -1, 'align_corners:1': -1, 'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_trilinear_fwd_packed': {
        'packed:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'alpha_range:null': -1,
        'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1,
        'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'slab:-1': -1,
    },
    'b200drr_trilinear_fwd_packed_v16': {
        'packed:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'alpha_range:null': -1,
        'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1,
        'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'slab:-1': -1, 'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_trilinear_fwd_sens_packed': {
        'packed:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1,
        'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1,
        'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'slab:-1': -1,
    },
    'b200drr_trilinear_fwd_sens_packed_v16': {
        'packed:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'out:null': -1, 'sens:null': -1,
        'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'H:0': -1,
        'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'slab:-1': -1,
        'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_trilinear_fwd_sens_pose': {
        'packed:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1, 'out:null': -1,
        'sens:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1,
        'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'slab:-1': -1,
    },
    'b200drr_trilinear_fwd_sens_pose_v16': {
        'packed:null': -1, 'src:null': -1, 'G:null': -1, 'Wd:null': -1, 'rows:null': -1, 'cols:null': -1, 'out:null': -1,
        'sens:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1,
        'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'n_points:1': -1, 'slab:-1': -1,
        'vol_type:0': -1, 'vol_type:3': -1,
    },
    'b200drr_polyrigid_fwd': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'M:null': -1, 'weights:null': -1, 'weights:+4': -1,
        'out:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1,
        'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1, 'H:-1': -1, 'H:1': -1, 'W:0': -1,
        'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1, 'K:0': -1, 'K:9': -2,
        'Bm:0': -1, 'Bm:3': -1, 'n_points:1': -1, 'packed:set': -1, 'packed:only+4': -1, 'too_big': -2, 'lattice_too_big': -2,
        'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&packed:only+4': -1, 'too_big&weights:+4': -1,
        'too_big&Bm:3': -1, 'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1,
        'lattice_too_big&packed:only+4': -1, 'lattice_too_big&weights:+4': -1, 'lattice_too_big&Bm:3': -1,
        'lattice_too_big&n_points:1': -1, 'K:9&vol:null': -1, 'K:9&B:65536': -1, 'K:9&packed:only+4': -1, 'K:9&weights:+4': -1,
        'K:9&Bm:3': -1, 'K:9&n_points:1': -1,
    },
    'b200drr_polyrigid_fwd_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'M:null': -1, 'weights:null': -1, 'weights:+4': -1,
        'out:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1,
        'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1, 'H:-1': -1, 'H:1': -1, 'W:0': -1,
        'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1, 'K:0': -1, 'K:9': -2,
        'Bm:0': -1, 'Bm:3': -1, 'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'packed:set': -1, 'packed:only+4': -1,
        'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
        'too_big&packed:only+4': -1, 'too_big&weights:+4': -1, 'too_big&Bm:3': -1, 'too_big&n_points:1': -1,
        'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1, 'lattice_too_big&vol_type:0': -1,
        'lattice_too_big&packed:only+4': -1, 'lattice_too_big&weights:+4': -1, 'lattice_too_big&Bm:3': -1,
        'lattice_too_big&n_points:1': -1, 'K:9&vol:null': -1, 'K:9&B:65536': -1, 'K:9&vol_type:0': -1, 'K:9&packed:only+4': -1,
        'K:9&weights:+4': -1, 'K:9&Bm:3': -1, 'K:9&n_points:1': -1,
    },
    'b200drr_polyrigid_bwd': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'M:null': -1, 'weights:null': -1, 'weights:+4': -1,
        'gout:null': -1, 'scratch:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1,
        'D2:0': -1, 'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1,
        'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1,
        'N:5': -1, 'K:0': -1, 'K:9': -2, 'Bm:0': -1, 'Bm:3': -1, 'n_points:1': -1, 'packed:set': -1, 'packed:only+4': -1,
        'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&packed:only+4': -1,
        'too_big&weights:+4': -1, 'too_big&Bm:3': -1, 'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1,
        'lattice_too_big&B:65536': -1, 'lattice_too_big&packed:only+4': -1, 'lattice_too_big&weights:+4': -1,
        'lattice_too_big&Bm:3': -1, 'lattice_too_big&n_points:1': -1, 'K:9&vol:null': -1, 'K:9&B:65536': -1,
        'K:9&packed:only+4': -1, 'K:9&weights:+4': -1, 'K:9&Bm:3': -1, 'K:9&n_points:1': -1,
    },
    'b200drr_polyrigid_bwd_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'M:null': -1, 'weights:null': -1, 'weights:+4': -1,
        'gout:null': -1, 'scratch:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1,
        'D2:0': -1, 'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1,
        'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1,
        'N:5': -1, 'K:0': -1, 'K:9': -2, 'Bm:0': -1, 'Bm:3': -1, 'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1,
        'packed:set': -1, 'packed:only+4': -1, 'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1,
        'too_big&B:65536': -1, 'too_big&vol_type:0': -1, 'too_big&packed:only+4': -1, 'too_big&weights:+4': -1,
        'too_big&Bm:3': -1, 'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1,
        'lattice_too_big&vol_type:0': -1, 'lattice_too_big&packed:only+4': -1, 'lattice_too_big&weights:+4': -1,
        'lattice_too_big&Bm:3': -1, 'lattice_too_big&n_points:1': -1, 'K:9&vol:null': -1, 'K:9&B:65536': -1,
        'K:9&vol_type:0': -1, 'K:9&packed:only+4': -1, 'K:9&weights:+4': -1, 'K:9&Bm:3': -1, 'K:9&n_points:1': -1,
    },
    'b200drr_polyrigid_jac': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'M:null': -1, 'weights:null': -1, 'weights:+4': -1,
        'T:null': -1, 'img:null': -1, 'J:null': -1, 'rects:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1,
        'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1,
        'g2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'K:0': -1, 'K:9': -2,
        'Bm:0': -1, 'Bm:3': -1, 'n_points:1': -1, 'packed:set': -1, 'packed:only+4': -1, 'too_big': -2, 'lattice_too_big': -2,
        'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&packed:only+4': -1, 'too_big&weights:+4': -1,
        'too_big&Bm:3': -1, 'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1,
        'lattice_too_big&packed:only+4': -1, 'lattice_too_big&weights:+4': -1, 'lattice_too_big&Bm:3': -1,
        'lattice_too_big&n_points:1': -1, 'K:9&vol:null': -1, 'K:9&B:65536': -1, 'K:9&packed:only+4': -1, 'K:9&weights:+4': -1,
        'K:9&Bm:3': -1, 'K:9&n_points:1': -1,
    },
    'b200drr_polyrigid_jac_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'M:null': -1, 'weights:null': -1, 'weights:+4': -1,
        'T:null': -1, 'img:null': -1, 'J:null': -1, 'rects:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1,
        'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1,
        'g2:-1': -1, 'H:0': -1, 'H:-1': -1, 'W:0': -1, 'W:-1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'K:0': -1, 'K:9': -2,
        'Bm:0': -1, 'Bm:3': -1, 'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'packed:set': -1, 'packed:only+4': -1,
        'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
        'too_big&packed:only+4': -1, 'too_big&weights:+4': -1, 'too_big&Bm:3': -1, 'too_big&n_points:1': -1,
        'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1, 'lattice_too_big&vol_type:0': -1,
        'lattice_too_big&packed:only+4': -1, 'lattice_too_big&weights:+4': -1, 'lattice_too_big&Bm:3': -1,
        'lattice_too_big&n_points:1': -1, 'K:9&vol:null': -1, 'K:9&B:65536': -1, 'K:9&vol_type:0': -1, 'K:9&packed:only+4': -1,
        'K:9&weights:+4': -1, 'K:9&Bm:3': -1, 'K:9&n_points:1': -1,
    },
    'b200drr_deform_fwd': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'field:null': -1, 'field:+4': -1, 'out:null': -1,
        'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'g0:0': -1,
        'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1, 'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1,
        'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1, 'Bf:0': -1, 'Bf:3': -1,
        'n_points:1': -1, 'packed:set': -1, 'packed:only+4': -1, 'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1,
        'too_big&B:65536': -1, 'too_big&packed:only+4': -1, 'too_big&field:+4': -1, 'too_big&Bf:3': -1,
        'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1,
        'lattice_too_big&packed:only+4': -1, 'lattice_too_big&field:+4': -1, 'lattice_too_big&Bf:3': -1,
        'lattice_too_big&n_points:1': -1,
    },
    'b200drr_deform_fwd_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'field:null': -1, 'field:+4': -1, 'out:null': -1,
        'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1, 'D2:-1': -1, 'g0:0': -1,
        'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1, 'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1,
        'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1, 'Bf:0': -1, 'Bf:3': -1,
        'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'packed:set': -1, 'packed:only+4': -1, 'too_big': -2,
        'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
        'too_big&packed:only+4': -1, 'too_big&field:+4': -1, 'too_big&Bf:3': -1, 'too_big&n_points:1': -1,
        'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1, 'lattice_too_big&vol_type:0': -1,
        'lattice_too_big&packed:only+4': -1, 'lattice_too_big&field:+4': -1, 'lattice_too_big&Bf:3': -1,
        'lattice_too_big&n_points:1': -1,
    },
    'b200drr_deform_bwd': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'field:null': -1, 'field:+4': -1, 'gout:null': -1,
        'g_field:+4': -1, 'scratch:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1,
        'D2:0': -1, 'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1,
        'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1,
        'N:5': -1, 'Bf:0': -1, 'Bf:3': -1, 'n_points:1': -1, 'packed:set': -1, 'packed:only+4': -1, 'too_big': -2,
        'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&packed:only+4': -1,
        'too_big&field:+4': -1, 'too_big&g_field:+4': -1, 'too_big&Bf:3': -1, 'too_big&n_points:1': -1,
        'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1, 'lattice_too_big&packed:only+4': -1,
        'lattice_too_big&field:+4': -1, 'lattice_too_big&g_field:+4': -1, 'lattice_too_big&Bf:3': -1,
        'lattice_too_big&n_points:1': -1,
    },
    'b200drr_deform_bwd_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'field:null': -1, 'field:+4': -1, 'gout:null': -1,
        'g_field:+4': -1, 'scratch:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1,
        'D2:0': -1, 'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1,
        'H:-1': -1, 'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1,
        'N:5': -1, 'Bf:0': -1, 'Bf:3': -1, 'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'packed:set': -1,
        'packed:only+4': -1, 'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1,
        'too_big&vol_type:0': -1, 'too_big&packed:only+4': -1, 'too_big&field:+4': -1, 'too_big&g_field:+4': -1,
        'too_big&Bf:3': -1, 'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1,
        'lattice_too_big&vol_type:0': -1, 'lattice_too_big&packed:only+4': -1, 'lattice_too_big&field:+4': -1,
        'lattice_too_big&g_field:+4': -1, 'lattice_too_big&Bf:3': -1, 'lattice_too_big&n_points:1': -1,
    },
    'b200drr_deform_jvp': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'field:null': -1, 'field:+4': -1, 'tangent:null': -1,
        'tangent:+4': -1, 'jv:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1, 'H:-1': -1,
        'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1,
        'Bf:0': -1, 'Bf:3': -1, 'n_points:1': -1, 'packed:set': -1, 'packed:only+4': -1, 'too_big': -2, 'lattice_too_big': -2,
        'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&packed:only+4': -1, 'too_big&field:+4': -1,
        'too_big&tangent:+4': -1, 'too_big&Bf:3': -1, 'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1,
        'lattice_too_big&B:65536': -1, 'lattice_too_big&packed:only+4': -1, 'lattice_too_big&field:+4': -1,
        'lattice_too_big&tangent:+4': -1, 'lattice_too_big&Bf:3': -1, 'lattice_too_big&n_points:1': -1,
    },
    'b200drr_deform_jvp_v16': {
        'vol:null': -1, 'src:null': -1, 'tgt:null': -1, 'raylen:null': -1, 'field:null': -1, 'field:+4': -1, 'tangent:null': -1,
        'tangent:+4': -1, 'jv:null': -1, 'alpha_range:null': -1, 'D0:0': -1, 'D0:-1': -1, 'D1:0': -1, 'D1:-1': -1, 'D2:0': -1,
        'D2:-1': -1, 'g0:0': -1, 'g0:-1': -1, 'g1:0': -1, 'g1:-1': -1, 'g2:0': -1, 'g2:-1': -1, 'H:0': -1, 'H:-1': -1,
        'H:1': -1, 'W:0': -1, 'W:-1': -1, 'W:1': -1, 'B:0': -1, 'B:-1': -1, 'B:65536': -1, 'N:0': -1, 'N:-1': -1, 'N:5': -1,
        'Bf:0': -1, 'Bf:3': -1, 'n_points:1': -1, 'vol_type:0': -1, 'vol_type:3': -1, 'packed:set': -1, 'packed:only+4': -1,
        'too_big': -2, 'lattice_too_big': -2, 'too_big&vol:null': -1, 'too_big&B:65536': -1, 'too_big&vol_type:0': -1,
        'too_big&packed:only+4': -1, 'too_big&field:+4': -1, 'too_big&tangent:+4': -1, 'too_big&Bf:3': -1,
        'too_big&n_points:1': -1, 'lattice_too_big&vol:null': -1, 'lattice_too_big&B:65536': -1,
        'lattice_too_big&vol_type:0': -1, 'lattice_too_big&packed:only+4': -1, 'lattice_too_big&field:+4': -1,
        'lattice_too_big&tangent:+4': -1, 'lattice_too_big&Bf:3': -1, 'lattice_too_big&n_points:1': -1,
    },
}

def test_refusal_codes_match_the_table():
    from diffdrr_b200 import build as b200build

    b200build.build()
    assert set(EXPECTED) == {_entry(n, t) for n in PAIRS for t in (False, True)}
    assert all(c in (EINVAL, EUNSUPPORTED) for codes in EXPECTED.values() for c in codes.values())
    got = _in_child({e: list(codes) for e, codes in EXPECTED.items()})
    bad = [f"{e} {label}: expected {c}, got {got[e][label]}" for e, codes in EXPECTED.items() for label, c in codes.items()
           if got[e][label] != c]
    assert not bad, f"{len(bad)} refusal codes changed:\n" + "\n".join(bad[:50])


if __name__ == "__main__":
    table = _record()
    print("EXPECTED = {")
    for e, codes in table.items():
        print(f"    {e!r}: {{")
        line = "       "
        for label, c in codes.items():
            item = f" {label!r}: {c},"
            if len(line) + len(item) > 128:
                print(line)
                line = "       "
            line += item
        print(line)
        print("    },")
    print("}")
