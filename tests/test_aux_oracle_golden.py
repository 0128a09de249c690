"""The auxiliary oracle (navigation-task epilogue, IMU) against fixtures produced by the reference's own code."""
import os

import numpy as np
import torch

from oracle import aux_oracle as A

G = os.path.join(os.path.dirname(__file__), "golden")


def _t(x):
    return torch.tensor(np.asarray(x))


def test_nav_reward_matches_reference():
    d = np.load(os.path.join(G, "nav_task_epilogue.npz"))
    assert tuple(d["param_names"]) == A.NAV_PARAM_NAMES
    p = {k: float(v) for k, v in zip(d["param_names"], d["param_values"])}
    err = A.nav_pos_error(_t(d["vehicle_orientation"]), _t(d["target"]), _t(d["pos"]))
    assert torch.allclose(err, _t(d["pos_error"]), rtol=0, atol=2e-6)
    for tag in ("c0", "c1"):
        r = A.nav_compute_reward(_t(d["pos_error"]), _t(d["prev_pos_error"]), _t(d["crashes"]), _t(d["actions"]), _t(d["prev_actions"]),
                                 float(d[f"frac_{tag}"]), p)
        ref = _t(d[f"reward_{tag}"])
        assert torch.allclose(r, ref, rtol=1e-6, atol=2e-5), (r - ref).abs().max()
        assert (r[_t(d["crashes"])] == -100.0).all()


def test_nav_obs_matches_reference():
    d = np.load(os.path.join(G, "nav_task_epilogue.npz"))
    obs = A.nav_process_obs(_t(d["vehicle_orientation"]), _t(d["pos"]), _t(d["target"]), _t(d["euler"]), _t(d["body_linvel"]),
                            _t(d["body_angvel"]), _t(d["robot_actions"]), _t(d["obs_draw_vec"]), _t(d["obs_draw_euler"]))
    ref = _t(d["obs"])
    assert torch.allclose(obs, ref[:, :17], rtol=1e-6, atol=2e-6), (obs - ref[:, :17]).abs().max()
    assert (ref[:, 17:] == 7.0).all()  # latents untouched without the VAE


def test_imu_matches_reference():
    d = np.load(os.path.join(G, "imu_sensor.npz"))
    grav = torch.tensor([0.0, 0.0, -9.81])
    for tag in ("body", "world", "gcomp"):
        wf, gc = bool(d[f"{tag}_cfg"][0]), bool(d[f"{tag}_cfg"][1])
        bias = _t(d[f"{tag}_bias0"])
        draws = _t(d[f"{tag}_draws"])
        for k in range(3):
            meas, bias = A.imu_update(_t(d[f"{tag}_force_sensor_tensor"]), _t(d[f"{tag}_robot_mass"]), _t(d[f"{tag}_robot_orientation"]),
                                      _t(d[f"{tag}_robot_body_angvel"]), _t(d[f"{tag}_sensor_quats"]), grav, wf, gc, bias,
                                      draws[2 * k], draws[2 * k + 1], _t(d["imu_noise_std"]).float(), _t(d["bias_std"]).float(),
                                      _t(d["max_measurement_value"]).float(), 0.01)
            ref = _t(d[f"{tag}_meas"][k])
            assert torch.allclose(meas, ref, rtol=1e-6, atol=1e-5), (tag, k, (meas - ref).abs().max())
        assert torch.allclose(bias, _t(d[f"{tag}_bias_end"]), rtol=1e-6, atol=1e-9)
        assert (meas.abs()[:, :3] <= 100.0).all() and (meas[:3, :3].abs() == 100.0).any()  # the clamp was exercised


def test_vae_encoder_equals_reference_encoder():
    """utils/vae_encoder.py loads the reference checkpoint and reproduces the reference encoder bit for bit
    (runs only where AERIAL_GYM_REFERENCE names a reference checkout: the 44 MB checkpoint is not part of this repository)."""
    import contextlib
    import io
    import sys

    import pytest

    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import _ref_loader

    wdir = os.path.join(_ref_loader.REF_ROOT, "aerial_gym/utils/vae/weights")
    if not os.path.isdir(wdir):
        pytest.skip("reference tree (with the VAE checkpoint) not present")
    _ref_loader.install()
    with contextlib.redirect_stdout(io.StringIO()):
        from aerial_gym.utils.vae.VAE import VAE
        ref = VAE(input_dim=1, latent_dim=64)
    from aerial_gym_simulator_b200.config.task_config import navigation_task_config
    from aerial_gym_simulator_b200.utils.vae_encoder import VAEImageEncoder

    class V(navigation_task_config.vae_config):
        model_folder = wdir
    ours = VAEImageEncoder(V, device="cpu")
    assert ours.weights_loaded
    sd = torch.load(os.path.join(wdir, V.model_file), map_location="cpu")
    ref.load_state_dict({k.replace("module.", "").replace("dronet.", "encoder."): v for k, v in sd.items()})
    ref.eval()
    x = torch.rand(2, 1, 270, 480, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        assert torch.equal(ref.encoder(x), ours.encoder(x))
