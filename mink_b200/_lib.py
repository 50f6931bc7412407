"""ctypes binding of libbik.so (include/bik.h).  No fallback: a missing library is an error."""

from __future__ import annotations

import ctypes as C
import os

from ._abi import BikBounds, BikCollision, BikDims, BikFrame, BikInputs, BikLimitDesc, BikTaskDesc

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libbik.so")
_lib = None

EXPORTS = ["bik_version", "bik_last_error", "bik_model_create", "bik_model_destroy", "bik_problem_create",
           "bik_problem_destroy", "bik_problem_dims", "bik_fk", "bik_frame_jacobian", "bik_fk_jac",
           "bik_qp_objective", "bik_limits_box", "bik_solve", "bik_solve_ex", "bik_integrate", "bik_check_limits", "bik_step",
           "bik_step_host", "bik_workspace_bytes", "bik_problem_describe", "bik_converge", "bik_track",
           "bik_fk64", "bik_frame_jacobian64", "bik_fk_jac64", "bik_qp_objective64", "bik_limits_box64", "bik_solve64",
           "bik_integrate64", "bik_check_limits64", "bik_step64", "bik_converge64", "bik_track64", "bik_measure_fma_peak",
           "bik_step_weighted", "bik_converge_weighted", "bik_track_weighted", "bik_step_weighted64", "bik_converge_weighted64",
           "bik_track_weighted64", "bik_step_weighted_ex", "bik_converge_weighted_ex", "bik_track_weighted_ex",
           "bik_step_weighted_ex64", "bik_converge_weighted_ex64", "bik_track_weighted_ex64", "bik_step_bounded",
           "bik_converge_bounded", "bik_track_bounded", "bik_step_bounded64", "bik_converge_bounded64", "bik_track_bounded64",
           "bik_step_coll", "bik_converge_coll", "bik_track_coll", "bik_step_coll64", "bik_converge_coll64", "bik_track_coll64",
           "bik_track_hold", "bik_track_hold64", "bik_step_placed", "bik_converge_placed", "bik_track_placed",
           "bik_step_placed64", "bik_converge_placed64", "bik_track_placed64"]


class BikError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libbik error {code}: {message}")
        self.code, self.message = code, message


def lib_path() -> str:
    return _LIB_PATH


def load():
    """Load libbik.so.  Raises if it has not been built (`python -m mink_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(f"{_LIB_PATH} is missing: build it with `python -m mink_b200.build` "
                           "(there is no CPU/PyTorch fallback for the IK hot path)")
    lib = C.CDLL(_LIB_PATH)
    vp, ci, cf, cd = C.c_void_p, C.c_int, C.c_float, C.c_double
    lib.bik_version.restype = ci
    lib.bik_last_error.restype = C.c_char_p
    lib.bik_model_create.argtypes = [vp, C.c_size_t, ci, C.POINTER(vp)]
    lib.bik_model_destroy.argtypes = [vp]
    lib.bik_model_destroy.restype = None
    lib.bik_problem_create.argtypes = [vp, C.POINTER(BikTaskDesc), ci, C.POINTER(BikLimitDesc), ci, C.POINTER(vp)]
    lib.bik_problem_destroy.argtypes = [vp]
    lib.bik_problem_destroy.restype = None
    lib.bik_problem_dims.argtypes = [vp, C.POINTER(BikDims)]
    lib.bik_fk.argtypes = [vp, ci, vp, C.POINTER(BikFrame), ci, vp, vp, vp]
    lib.bik_frame_jacobian.argtypes = [vp, ci, vp, C.POINTER(BikFrame), ci, vp, vp]
    lib.bik_fk_jac.argtypes = [vp, ci, C.POINTER(BikInputs), cf, vp, vp, vp, vp, vp, vp]
    lib.bik_qp_objective.argtypes = [vp, ci, vp, vp, vp, cd, vp, vp, vp]
    lib.bik_limits_box.argtypes = [vp, ci, vp, cf, vp, vp, vp]
    lib.bik_solve.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, cf, cd, vp, vp, vp]
    lib.bik_solve_ex.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, cf, cd, vp, vp, vp, vp]
    lib.bik_integrate.argtypes = [vp, ci, vp, vp, vp]
    lib.bik_check_limits.argtypes = [vp, ci, vp, cf, vp, vp]
    lib.bik_step.argtypes = [vp, ci, vp, C.POINTER(BikInputs), cf, cd, ci, ci, vp, vp, vp]
    lib.bik_step_host.argtypes = [vp, ci, vp, C.POINTER(BikInputs), cf, cd, ci, ci, vp, vp,
                                  C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.bik_workspace_bytes.argtypes = [vp, ci]
    lib.bik_workspace_bytes.restype = C.c_size_t
    lib.bik_converge.argtypes = [vp, ci, vp, C.POINTER(BikInputs), cf, cd, ci, cf, cf, ci, vp, vp, vp]
    lib.bik_track.argtypes = [vp, ci, ci, vp, C.POINTER(BikInputs), vp, cf, cd, ci, cf, cf, ci, vp, vp, vp, vp, vp]
    lib.bik_problem_describe.argtypes = [vp, cd, C.c_char_p, C.c_size_t]
    # fp64 mirror (double buffers, bik_inputs.f64 = 1)
    lib.bik_fk64.argtypes = lib.bik_fk.argtypes
    lib.bik_frame_jacobian64.argtypes = lib.bik_frame_jacobian.argtypes
    lib.bik_fk_jac64.argtypes = [vp, ci, C.POINTER(BikInputs), cd, vp, vp, vp, vp, vp, vp]
    lib.bik_qp_objective64.argtypes = lib.bik_qp_objective.argtypes
    lib.bik_limits_box64.argtypes = [vp, ci, vp, cd, vp, vp, vp]
    lib.bik_solve64.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, cd, cd, vp, vp, vp, vp]
    lib.bik_integrate64.argtypes = lib.bik_integrate.argtypes
    lib.bik_check_limits64.argtypes = [vp, ci, vp, cd, vp, vp]
    lib.bik_step64.argtypes = [vp, ci, vp, C.POINTER(BikInputs), cd, cd, ci, ci, vp, vp, vp]
    lib.bik_converge64.argtypes = [vp, ci, vp, C.POINTER(BikInputs), cd, cd, ci, cd, cd, ci, vp, vp, vp]
    lib.bik_track64.argtypes = [vp, ci, ci, vp, C.POINTER(BikInputs), vp, cd, cd, ci, cd, cd, ci, vp, vp, vp, vp, vp]
    lib.bik_measure_fma_peak.argtypes = [ci, ci, ci, C.POINTER(cd)]
    # per-instance task weights: the same arguments with the weights pointer after the inputs
    for name in ("bik_step", "bik_converge", "bik_track", "bik_step64", "bik_converge64", "bik_track64"):
        args = getattr(lib, name).argtypes
        at = args.index(C.POINTER(BikInputs)) + 1
        getattr(lib, name.replace("64", "") + "_weighted" + ("64" if name.endswith("64") else "")).argtypes = args[:at] + [vp] + args[at:]
        # per-instance posture weights: one more pointer after the task weights
        getattr(lib, name.replace("64", "") + "_weighted_ex" + ("64" if name.endswith("64") else "")).argtypes = args[:at] + [vp, vp] + args[at:]
        # per-instance bounds: a bik_bounds after the posture weights
        getattr(lib, name.replace("64", "") + "_bounded" + ("64" if name.endswith("64") else "")).argtypes = (args[:at] + [vp, vp, C.POINTER(BikBounds)]
                                                                                                     + args[at:])
        # per-instance collision pairs and distances: a bik_collision after the bounds
        getattr(lib, name.replace("64", "") + "_coll" + ("64" if name.endswith("64") else "")).argtypes = (
            args[:at] + [vp, vp, C.POINTER(BikBounds), C.POINTER(BikCollision)] + args[at:])
    # held targets (bik_track only): the hold mask after the collision arguments
    for name in ("bik_track_coll", "bik_track_coll64"):
        args = getattr(lib, name).argtypes
        at = args.index(C.POINTER(BikCollision)) + 1
        getattr(lib, name.replace("_coll", "_hold")).argtypes = args[:at] + [vp] + args[at:]
    # per-instance frame placement: the placement rows after the collision arguments (bik_track: after the hold mask)
    for name in ("bik_step_coll", "bik_converge_coll", "bik_step_coll64", "bik_converge_coll64", "bik_track_hold", "bik_track_hold64"):
        args = getattr(lib, name).argtypes
        at = args.index(C.POINTER(BikCollision)) + (2 if "_hold" in name else 1)
        getattr(lib, name.replace("_coll", "_placed").replace("_hold", "_placed")).argtypes = args[:at] + [vp] + args[at:]
    _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        raise BikError(rc, load().bik_last_error().decode(errors="replace"))
