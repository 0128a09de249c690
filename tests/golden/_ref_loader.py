"""Import the *reference's own* torch control stack on CPU.

Test infrastructure, never imported by the product.  The reference is a checkout of
ntnu-arl/aerial_gym_simulator (commit f0d0f05) named by the ``AERIAL_GYM_REFERENCE``
environment variable; it is not part of this repository.  This module is used by
``tests/golden/make_golden*.py`` to produce the committed fixtures and by the
optional ``-m "not gpu"`` cross-checks that skip when no reference is given.

Procedure (SURVEY.md section 8c): register ``aerial_gym`` as a namespace module
whose ``__path__`` points into the reference tree (this skips the package
``__init__`` that imports isaacgym and every task), register empty
``isaacgym.*`` modules and a ``pytorch3d.transforms`` stub whose two functions
restate the published pytorch3d algorithms.
"""
import os
import sys
import types

import torch

REF_ROOT = os.environ.get("AERIAL_GYM_REFERENCE", "")


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "aerial_gym", "control"))


def _matrix_to_quaternion(matrix: torch.Tensor) -> torch.Tensor:
    """Published pytorch3d algorithm (pytorch3d/transforms/rotation_conversions.py):
    four candidate quaternions, pick the one with the largest denominator.
    Returns (w, x, y, z)."""
    m = matrix
    m00, m01, m02 = m[..., 0, 0], m[..., 0, 1], m[..., 0, 2]
    m10, m11, m12 = m[..., 1, 0], m[..., 1, 1], m[..., 1, 2]
    m20, m21, m22 = m[..., 2, 0], m[..., 2, 1], m[..., 2, 2]

    def _sqrt_pos(x):
        out = torch.zeros_like(x)
        pos = x > 0
        out[pos] = torch.sqrt(x[pos])
        return out

    q_abs = _sqrt_pos(
        torch.stack(
            [1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22],
            dim=-1,
        )
    )
    quat_by_rijk = torch.stack(
        [
            torch.stack([q_abs[..., 0] ** 2, m21 - m12, m02 - m20, m10 - m01], dim=-1),
            torch.stack([m21 - m12, q_abs[..., 1] ** 2, m10 + m01, m02 + m20], dim=-1),
            torch.stack([m02 - m20, m10 + m01, q_abs[..., 2] ** 2, m12 + m21], dim=-1),
            torch.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[..., 3] ** 2], dim=-1),
        ],
        dim=-2,
    )
    flr = torch.tensor(0.1).to(dtype=q_abs.dtype)
    cand = quat_by_rijk / (2.0 * q_abs[..., None].max(flr))
    idx = q_abs.argmax(dim=-1)
    out = cand[torch.arange(cand.shape[0]), idx]
    return out


def _quaternion_to_matrix(q: torch.Tensor) -> torch.Tensor:
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack(
        (
            1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
            two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
            two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j),
        ),
        -1,
    )
    return o.reshape(q.shape[:-1] + (3, 3))


def install():
    """Make ``import aerial_gym.control`` etc. resolve into the reference tree."""
    if not reference_available():
        raise RuntimeError("reference tree not present")
    if "aerial_gym" in sys.modules and getattr(sys.modules["aerial_gym"], "_b200_ref_stub", False):
        return
    pkg = types.ModuleType("aerial_gym")
    pkg.__path__ = [os.path.join(REF_ROOT, "aerial_gym")]
    pkg.AERIAL_GYM_DIRECTORY = REF_ROOT
    pkg._b200_ref_stub = True
    sys.modules["aerial_gym"] = pkg
    for name in ("isaacgym", "isaacgym.gymapi", "isaacgym.gymutil", "isaacgym.gymtorch"):
        sys.modules.setdefault(name, types.ModuleType(name))
    p3d = types.ModuleType("pytorch3d")
    p3dt = types.ModuleType("pytorch3d.transforms")
    p3dt.matrix_to_quaternion = _matrix_to_quaternion
    p3dt.quaternion_to_matrix = _quaternion_to_matrix
    p3d.transforms = p3dt
    sys.modules["pytorch3d"] = p3d
    sys.modules["pytorch3d.transforms"] = p3dt
