import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_addoption(parser):
    parser.addoption("--gpu-dryrun", action="store_true", default=False,
                     help="run the TEXT of -m gpu tests on CPU: module-level DEV -> 'cpu', the C-ABI entry points of the small kernels -> "
                          "their host shadows, engine / ray-caster -> the CPU twins (tests/_cpu_stack.py).  Finds mistakes in test code "
                          "written without a GPU; proves nothing about the kernels' thread mapping.")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    """GPU tests fail loudly (not skip) when selected on a box without CUDA: a silent skip
    would hide a missing native path.  Each one gets a wall-clock limit (pytest-timeout, where installed): a kernel that
    never returns must end the run with a failure, not hold the GPU box until the driver's own limit."""
    if not config.pluginmanager.hasplugin("timeout"):
        return
    for item in items:
        if item.get_closest_marker("gpu") is not None and item.get_closest_marker("timeout") is None:
            item.add_marker(pytest.mark.timeout(900))


@pytest.fixture(autouse=True)
def _gpu_dryrun(request, monkeypatch):
    if not request.config.getoption("--gpu-dryrun") or request.node.get_closest_marker("gpu") is None:
        yield
        return
    import torch

    from ._cpu_stack import cpu_stack
    import importlib

    from . import _cpu_stack as CS
    twins = {"DEV": "cpu", "RayScene": CS.CpuRayScene, "RaySensor": CS.CpuRaySensor, "DeviceSensorNoise": CS.CpuDeviceSensorNoise,
             "Hp1Engine": CS.CpuHp1Engine}
    for mod in (request.module, importlib.import_module("tests.test_hp2_gpu")):  # (the zz tests borrow test_hp2_gpu's scene builders)
        for name, twin in twins.items():
            if hasattr(mod, name):
                monkeypatch.setattr(mod, name, twin)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    import aerial_gym_simulator_b200.task  # noqa: F401  (registers the tasks)
    from aerial_gym_simulator_b200.registry._core import task_registry
    for cfg in set(task_registry.get_task_configs().values() if isinstance(task_registry.get_task_configs(), dict) else task_registry.get_task_configs()):
        if isinstance(getattr(cfg, "device", None), str):
            monkeypatch.setattr(cfg, "device", "cpu")
    with cpu_stack():
        yield
