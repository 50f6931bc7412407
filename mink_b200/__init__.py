"""mink_b200 -- batched differential inverse kinematics on NVIDIA H100 behind mink's Python API.

Only the `solve_ik` hot path of kevinzakka/mink is rebuilt here (SURVEY.md section 8): FK + task
errors/Jacobians + QP assembly + exact active-set solve + integrate, as hand-written sm_90a kernels
in libbik.so (include/bik.h), driven through ctypes.  The names below mirror `mink/__init__.py:3-45`
for that path; see DESIGN.md and INTEGRATION.md.
"""

__version__ = "0.1.0"

from .exceptions import (InvalidDamping, InvalidFrame, InvalidGain, InvalidKeyframe, InvalidMocapBody, InvalidTarget,
                         LimitDefinitionError, MinkError, NotWithinConfigurationLimits, TargetNotSet,
                         TaskDefinitionError, UnsupportedFrame)
from .lie import SE3, SO3, MatrixLieGroup
from .mjcf import Model
from .flatten import FlatModel, flatten
from .utils import (custom_configuration_vector, get_body_body_ids, get_body_geom_ids, get_freejoint_dims,
                    get_subtree_body_ids, get_subtree_geom_ids)


def __getattr__(name):
    """Heavier symbols (they import torch) are resolved lazily."""
    import importlib

    table = {
        "Configuration": "configuration", "SUPPORTED_FRAMES": "configuration",
        "Task": "tasks", "Objective": "tasks", "FrameTask": "tasks", "PostureTask": "tasks", "DampingTask": "tasks",
        "ComTask": "tasks", "RelativeFrameTask": "tasks",
        "Limit": "limits", "Constraint": "limits", "ConfigurationLimit": "limits", "VelocityLimit": "limits",
        "CollisionAvoidanceLimit": "limits",
        "build_ik": "ik", "solve_ik": "ik", "converge_ik": "ik", "track_ik": "ik",
    }
    if name in table:
        return getattr(importlib.import_module(f"{__name__}.{table[name]}"), name)
    raise AttributeError(name)
