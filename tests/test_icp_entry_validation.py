"""Argument validation of the ICP entry points (icp.cu): every o3db_icp_create*, every one-shot o3db_icp_*, and the
handle calls.  Each rejected call must return its code and set its exact o3db_last_error() text, and the checks must
fire in their order, all before any CUDA call, so no GPU is needed.  With valid arguments and no device, every entry
point fails with ERR_CUDA: there is no CPU fallback."""
import ctypes as C

import numpy as np
import pytest
import torch

EMPTY = "Source and/or Target pointcloud is empty."
NULL_OPTIONS = "o3db_icp_create: null options / init"
NO_NORMALS = "Target pointcloud missing normals attribute."
SYM_NORMALS = "SymmetricICP requires both source and target to have normals."
DOP_NORMALS = "DopplerICP requires target pointcloud to have normals."
DOP_VALUES = "DopplerICP requires source pointcloud to have Doppler velocities."
DOP_DIRS = "DopplerICP requires source pointcloud to have pre-computed direction vectors."
LAMBDA = "lambda_geometric must be in [0, 1]"
DISTANCE = "max_correspondence_distance must be positive"
ITERATIONS = "max_iteration must be non-negative"

# parameter names of each entry point, in C order
PARAMS = {
    "o3db_icp_create": "src n tgt tgt_nrm m init opt comm stream out",
    "o3db_icp_create_colored": "src src_col n tgt tgt_nrm tgt_col tgt_grad m init opt lam comm stream out",
    "o3db_icp_create_point_to_point": "src n tgt m init opt comm stream out",
    "o3db_icp_create_symmetric": "src src_nrm n tgt tgt_nrm m init opt comm stream out",
    "o3db_icp_create_doppler": "src dop dirs n tgt tgt_nrm m init opt params comm stream out",
    "o3db_icp_point_to_plane": "src n tgt tgt_nrm m init opt result corr per stream",
    "o3db_icp_point_to_point": "src n tgt m init opt result corr per stream",
    "o3db_icp_symmetric": "src src_nrm n tgt tgt_nrm m init opt result corr per stream",
    "o3db_icp_doppler": "src dop dirs n tgt tgt_nrm m init opt params result corr per stream",
    "o3db_icp_colored": "src src_col n tgt tgt_nrm tgt_col tgt_grad m init opt lam result corr per stream",
    "o3db_icp_point_to_plane_host": "src n tgt tgt_nrm m init opt result corr per",
}
CREATE = [f for f in PARAMS if f.startswith("o3db_icp_create")]
ONE_SHOT = [f for f in PARAMS if not f.startswith("o3db_icp_create")]

_CASES = {   # (entry point, case name, overrides, code, message)
    "o3db_icp_create": [
        ("out", {"out": None}, "o3db_icp_create: out is null"),
    ],
    "o3db_icp_create_colored": [
        ("out", {"out": None}, "o3db_icp_create_colored: out is null"),
    ],
    "o3db_icp_create_point_to_point": [
        ("out", {"out": None}, "o3db_icp_create: out is null"),
    ],
    "o3db_icp_create_symmetric": [
        ("out", {"out": None}, "o3db_icp_create_symmetric: out is null"),
        ("comm", {"comm": "fake"}, "SymmetricICP does not run multi-GPU: pass no communicator."),
        ("comm_after_normals", {"comm": "fake", "src_nrm": None}, SYM_NORMALS),
        ("empty_before_comm", {"comm": "fake", "n": 0}, EMPTY),
        ("comm_before_options", {"comm": "fake", "opt": None}, "SymmetricICP does not run multi-GPU: pass no communicator."),
    ],
    "o3db_icp_create_doppler": [
        ("out", {"out": None}, "o3db_icp_create_doppler: out is null"),
        ("comm", {"comm": "fake"}, "DopplerICP does not run multi-GPU: pass no communicator."),
        ("comm_after_directions", {"comm": "fake", "dirs": None}, DOP_DIRS),
        ("params_after_comm", {"comm": "fake", "params": None}, "DopplerICP does not run multi-GPU: pass no communicator."),
        ("options_before_empty", {"opt": None, "n": 0}, NULL_OPTIONS),
    ],
}

# checks every entry point of an estimator shares with its create call
_SHARED = {
    "plane": [
        ("options", {"opt": None}, NULL_OPTIONS),
        ("init", {"init": None}, NULL_OPTIONS),
        ("source_null", {"src": None}, EMPTY),
        ("target_null", {"tgt": None}, EMPTY),
        ("source_empty", {"n": 0}, EMPTY),
        ("target_empty", {"m": 0}, EMPTY),
        ("normals", {"tgt_nrm": None}, NO_NORMALS),
        ("empty_before_normals", {"n": 0, "tgt_nrm": None}, EMPTY),
        ("options_before_empty", {"opt": None, "n": 0}, NULL_OPTIONS),
        ("too_many_points", {"n": 2**31 - 1 - 2048}, "o3db_icp_create: too many points"),
        ("distance", {"opt": "zero_distance"}, DISTANCE),
        ("iterations", {"opt": "negative_iterations"}, ITERATIONS),
    ],
    "colored": [
        ("options", {"opt": None}, NULL_OPTIONS),
        ("init", {"init": None}, NULL_OPTIONS),
        ("source_null", {"src": None}, EMPTY),
        ("target_empty", {"m": 0}, EMPTY),
        ("normals", {"tgt_nrm": None}, NO_NORMALS),
        ("source_colors", {"src_col": None}, "Source pointcloud missing colors attribute."),
        ("target_colors", {"tgt_col": None}, "Target pointcloud missing colors attribute."),
        ("gradients", {"tgt_grad": None},
         "Target pointcloud missing color_gradients attribute (o3db_estimate_color_gradients)."),
        ("lambda_below", {"lam": -0.1}, LAMBDA),
        ("lambda_above", {"lam": 1.1}, LAMBDA),
        ("lambda_nan", {"lam": float("nan")}, LAMBDA),
        ("colors_before_options", {"src_col": None, "opt": None}, "Source pointcloud missing colors attribute."),
        ("lambda_before_empty", {"lam": 2.0, "n": 0}, LAMBDA),
        ("distance", {"opt": "zero_distance"}, DISTANCE),
    ],
    "point": [
        ("options", {"opt": None}, NULL_OPTIONS),
        ("init", {"init": None}, NULL_OPTIONS),
        ("source_null", {"src": None}, EMPTY),
        ("target_empty", {"m": 0}, EMPTY),
        ("distance", {"opt": "zero_distance"}, DISTANCE),
        ("iterations", {"opt": "negative_iterations"}, ITERATIONS),
    ],
    "symmetric": [
        ("options", {"opt": None}, NULL_OPTIONS),
        ("init", {"init": None}, NULL_OPTIONS),
        ("source_null", {"src": None}, EMPTY),
        ("target_empty", {"m": 0}, EMPTY),
        ("source_normals", {"src_nrm": None}, SYM_NORMALS),
        ("target_normals", {"tgt_nrm": None}, SYM_NORMALS),
        ("empty_before_options", {"n": 0, "opt": None}, EMPTY),
        ("normals_before_options", {"src_nrm": None, "opt": None}, SYM_NORMALS),
        ("distance", {"opt": "zero_distance"}, DISTANCE),
    ],
    "doppler": [
        ("options", {"opt": None}, NULL_OPTIONS),
        ("init", {"init": None}, NULL_OPTIONS),
        ("source_null", {"src": None}, EMPTY),
        ("target_empty", {"m": 0}, EMPTY),
        ("normals", {"tgt_nrm": None}, DOP_NORMALS),
        ("dopplers", {"dop": None}, DOP_VALUES),
        ("directions", {"dirs": None}, DOP_DIRS),
        ("normals_first", {"tgt_nrm": None, "dop": None, "dirs": None}, DOP_NORMALS),
        ("params", {"params": None}, "DopplerICP: null parameters"),
        ("period", {"params": "short_period"}, "Time period too small."),
        ("kernel", {"params": "cauchy"}, "Unsupported method."),
        ("rotation", {"params": "singular"}, "DopplerICP: the rotation block of transform_vehicle_to_sensor is singular."),
        ("params_before_init", {"params": None, "init": None}, "DopplerICP: null parameters"),
        ("distance", {"opt": "zero_distance"}, DISTANCE),
    ],
}
_ESTIMATOR = {
    "o3db_icp_create": "plane", "o3db_icp_point_to_plane": "plane",
    "o3db_icp_create_colored": "colored", "o3db_icp_colored": "colored",
    "o3db_icp_create_point_to_point": "point", "o3db_icp_point_to_point": "point",
    "o3db_icp_create_symmetric": "symmetric", "o3db_icp_symmetric": "symmetric",
    "o3db_icp_create_doppler": "doppler", "o3db_icp_doppler": "doppler",
}
_HOST = [   # o3db_icp_point_to_plane_host checks its own arguments first, in this order
    ("source_null", {"src": None}, EMPTY),
    ("source_empty", {"n": 0}, EMPTY),
    ("target_empty", {"m": 0}, EMPTY),
    ("normals", {"tgt_nrm": None}, NO_NORMALS),
    ("options", {"opt": None}, "o3db_icp_point_to_plane_host: null options / result"),
    ("result", {"result": None}, "o3db_icp_point_to_plane_host: null options / result"),
    ("empty_before_normals", {"n": 0, "tgt_nrm": None}, EMPTY),
    ("normals_before_options", {"tgt_nrm": None, "opt": None}, NO_NORMALS),
]


def _cases():
    for fn in PARAMS:
        rows = _HOST if fn == "o3db_icp_point_to_plane_host" else _CASES.get(fn, []) + _SHARED[_ESTIMATOR[fn]]
        for name, over, msg in rows:
            yield pytest.param(fn, over, msg, id=f"{fn}-{name}")


class _Inputs:
    """Valid arguments for every entry point; host buffers stand in for the device ones, which no check reads."""

    def __init__(self):
        from open3d_b200 import _lib as L
        rng = np.random.default_rng(0)
        self.L = L
        self.pts = rng.uniform(-1, 1, (64, 3)).astype(np.float32)
        self.vals = rng.uniform(-1, 1, 64).astype(np.float32)
        self.eye = np.eye(4).ravel()
        self.per = np.zeros(16)
        self.corr = np.zeros(64, np.int64)
        self.fake = (C.c_char * 64)()   # a communicator no check may dereference
        self.result = L.IcpResult()
        self.out = C.c_void_p(0x1234)    # a failed create must null it

    def options(self, kind="valid"):
        L = self.L
        return L.IcpOptions(0.0 if kind == "zero_distance" else 0.2, -1 if kind == "negative_iterations" else 5, 0.0,
                            0.0, L.RobustKernel(0, 1.0, 1.0), 0.0)

    def params(self, kind="valid"):
        L = self.L
        T = [1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]
        if kind == "singular":
            T[0] = 0.0
        p = L.DopplerParams(1e-4 if kind == "short_period" else 0.1, 0.01, 0, 2.0, 2, 0, 2, L.RobustKernel(0, 1.0, 1.0),
                            L.RobustKernel(3 if kind == "cauchy" else 0, 1.0, 1.0), (C.c_double * 16)(*T))
        return p

    def args(self, fn, over):
        p, v = self.pts.ctypes.data, self.vals.ctypes.data
        a = dict(src=p, src_col=p, src_nrm=p, dop=v, dirs=p, n=64, tgt=p, tgt_nrm=p, tgt_col=p, tgt_grad=p, m=64,
                 init=self.eye.ctypes.data, opt="valid", lam=0.968, params="valid", comm=None, stream=None,
                 out=C.byref(self.out), result=C.byref(self.result), corr=self.corr.ctypes.data,
                 per=self.per.ctypes.data)
        a.update(over)
        if a["opt"] is not None:
            self.opt = self.options(a["opt"])
            a["opt"] = C.byref(self.opt)
        if a["params"] is not None:
            self.par = self.params(a["params"])
            a["params"] = C.byref(self.par)
        if a["comm"] == "fake":
            a["comm"] = C.addressof(self.fake)
        return [a[k] for k in PARAMS[fn].split()]


@pytest.mark.parametrize("fn, over, msg", list(_cases()))
def test_entry_point_rejects(fn, over, msg):
    x = _Inputs()
    rc = getattr(x.L.lib, fn)(*x.args(fn, over))
    assert (rc, x.L.last_error()) == (x.L.ERR_INVALID, msg)
    if fn in CREATE and over.get("out", 1) is not None:
        assert x.out.value is None


@pytest.mark.parametrize("fn, args, msg", [
    ("o3db_icp_reset", (None, None), "o3db_icp_reset: null handle"),
    ("o3db_icp_iterate", (None, 1, None), "o3db_icp_iterate: null handle"),
    ("o3db_icp_finish", (None, "result", None, None, None), "o3db_icp_finish: null argument"),
    ("o3db_icp_finish", (None, None, None, None, None), "o3db_icp_finish: null argument"),
    ("o3db_icp_state", (None, "result", None, None), "o3db_icp_state: null argument"),
    ("o3db_icp_state", (None, None, None, None), "o3db_icp_state: null argument"),
], ids=["reset", "iterate", "finish", "finish_no_result", "state", "state_no_result"])
def test_handle_calls_reject_null_handle(fn, args, msg):
    from open3d_b200 import _lib as L
    result = L.IcpResult()
    rc = getattr(L.lib, fn)(*[C.byref(result) if a == "result" else a for a in args])
    assert (rc, L.last_error()) == (L.ERR_INVALID, msg)


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
@pytest.mark.parametrize("fn", list(PARAMS))
def test_valid_arguments_fail_without_a_device(fn):
    x = _Inputs()
    rc = getattr(x.L.lib, fn)(*x.args(fn, {}))
    assert rc == x.L.ERR_CUDA and "cuda" in x.L.last_error().lower(), (rc, x.L.last_error())
    if fn in CREATE:
        assert x.out.value is None
