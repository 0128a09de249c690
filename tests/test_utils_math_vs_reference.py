"""utils/math.py mirror against the REFERENCE'S OWN utils/math.py on random inputs, function by function (this container only: the
test skips unless AERIAL_GYM_REFERENCE names a checkout of the reference).  Same names, same arguments, same values."""
import inspect
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import _ref_loader  # noqa: E402

pytestmark = pytest.mark.skipif(not _ref_loader.reference_available(), reason="reference tree not present")

from aerial_gym_simulator_b200.utils import math as M  # noqa: E402


def _ref():
    _ref_loader.install()
    from aerial_gym.utils import math as R
    return R


def _q(n, g):
    q = torch.randn(n, 4, generator=g)
    return q / q.norm(dim=1, keepdim=True)


def test_every_public_function_of_the_reference_exists():
    R = _ref()
    names = [n for n, f in vars(R).items() if not n.startswith("_") and (inspect.isfunction(f) or isinstance(f, torch.jit.ScriptFunction))
             and getattr(f, "__module__", "aerial_gym.utils.math") in ("aerial_gym.utils.math", None)]
    missing = [n for n in names if not hasattr(M, n) and n not in ("matrix_to_quaternion",)]  # (pytorch3d re-export)
    assert not missing, missing


def test_values_match_on_random_inputs():
    R = _ref()
    g = torch.Generator().manual_seed(0)
    n = 257
    q, q2, v, t = _q(n, g), _q(n, g), torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g)
    e = (torch.rand(n, 3, generator=g) * 2 - 1) * 3.0
    S = torch.randn(n, 3, 3, generator=g)
    S = S - S.transpose(1, 2)
    cases = {
        "quat_conjugate": (q,), "quat_inverse": (q,), "quat_mul": (q, q2), "quat_apply": (q, v), "quat_apply_inverse": (q, v),
        "quat_rotate": (q, v), "quat_rotate_inverse": (q, v), "quat_axis": (q, 2), "quat_from_euler_xyz": (e[:, 0], e[:, 1], e[:, 2]),
        "quat_from_euler_xyz_tensor": (e,), "get_euler_xyz_tensor": (q,), "ssa": (e * 3,), "vehicle_frame_quat_from_quat": (q,),
        "quat_to_rotation_matrix": (q,), "normalize": (v,), "tf_apply": (q, t, v), "tensor_clamp": (v, -torch.ones(3) * 0.5, torch.ones(3) * 0.5),
        "compute_vee_map": (S,), "scale": (v, torch.tensor(-2.0), torch.tensor(3.0)), "unscale": (v, torch.tensor(-2.0), torch.tensor(3.0)), "quat_unit": (q * 3,),
        "quat_from_angle_axis": (e[:, 0], v), "normalize_angle": (e * 4,), "tf_vector": (q, v), "get_basis_vector": (q, v),
        "pd_control": (v, t, torch.tensor(2.0), torch.tensor(0.5)), "copysign": (0.5 * np.pi, e[:, 0]), "torch_interpolate_ratio": (v, v + 2.0, torch.rand(n, 3, generator=g)),
        "exponential_reward_function": (2.0, 3.0, e[:, 0]), "exponential_penalty_function": (2.0, 3.0, e[:, 0]),
    }
    checked = 0
    for name, args in cases.items():
        if not hasattr(R, name):
            continue
        want, got = getattr(R, name)(*args), getattr(M, name)(*args)
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (name, (got - want).abs().max())
        checked += 1
    for name, args in (("tf_inverse", (q, t)), ("tf_combine", (q, t, q2, v))):
        for a, b in zip(getattr(M, name)(*args), getattr(R, name)(*args)):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), name
        checked += 1
    r, p, y = M.get_euler_xyz(q)
    rr, pp, yy = R.get_euler_xyz(q)
    assert torch.allclose(r, rr) and torch.allclose(p, pp) and torch.allclose(y, yy)
    # same generator stream, same arithmetic (the reference's TorchScript signatures: floats + (int, int) for the first, tensors +
    # (int, int, int) for the _vec one)
    torch.manual_seed(3)
    a = M.torch_rand_float(-1.5, 2.0, (n, 3), "cpu")
    torch.manual_seed(3)
    assert torch.equal(a, R.torch_rand_float(-1.5, 2.0, (n, 3), "cpu"))
    lo, hi = torch.tensor([-1.5, 0.0, 1.0]), torch.tensor([2.0, 0.5, 4.0])
    torch.manual_seed(3)
    a = M.torch_rand_float_vec(lo, hi, (n, 2, 3), "cpu")
    torch.manual_seed(3)
    assert torch.equal(a, R.torch_rand_float_vec(lo, hi, (n, 2, 3), "cpu"))
    torch.manual_seed(4)
    a = M.torch_rand_float_tensor(v, v + 1.0)
    torch.manual_seed(4)
    assert torch.equal(a, R.torch_rand_float_tensor(v, v + 1.0))
    torch.manual_seed(5)
    a = M.torch_random_dir_2((n, 1), "cpu")
    torch.manual_seed(5)
    assert torch.allclose(a, R.torch_random_dir_2((n, 1), "cpu"))
    assert checked >= 30
