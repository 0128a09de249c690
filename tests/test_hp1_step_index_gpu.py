"""The chained position-task step with its step index from the host (agx_hp1_position_task_step_at, what Hp1Engine calls) against
the same steps whose warps claim the index on the device (agx_hp1_position_task_step, for C callers that do not count their
launches): the same bits, and the same chain counters -- tile_sync's claim and done counts and any_reset[4:16].

The steps reuse eight action tensors, so after the first eight Hp1Engine.position_task_step takes its fast path, and the engine's
per-step output pointers are aimed at a new slot before every step: the fast path must launch with the live buffers."""
import ctypes as C

import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from tests.test_hp1_chained_gpu import K, assert_bits, chain_counters, engine, inputs, run

DEV = "cuda:0"


def device_claim(e):
    """e launches through the entry that claims the step index on the device"""
    lib = _lib.load()
    e._task_step_at = lambda cfg, buf, stream, T: lib.agx_hp1_position_task_step(C.byref(e.cfg), C.byref(e._buf), stream)
    return e


def count_full_path(e):
    """counts the calls that validate their actions tensor: the ones that did not take the fast path"""
    calls = [0]
    check = e._check_actions

    def counted(a):
        calls[0] += 1
        check(a)

    e._check_actions = counted
    return calls


@pytest.mark.gpu
@pytest.mark.parametrize("N", [777, 65536])
def test_host_step_index_equals_device_claim(N):
    spec, root, params, target, steps0, acts = inputs(N, "mix")
    seq = [acts[i % 8] for i in range(K)]
    ser = device_claim(engine(spec, N, root, params, target, steps0))
    assert ser._chain_counts
    ref = run(ser, seq)
    claimed = device_claim(engine(spec, N, root, params, target, steps0))
    assert_bits(ref, run(claimed, seq, overlapped=True), "device claim: overlapped vs serialised")
    assert_bits(chain_counters(ser), chain_counters(claimed), "device claim: chain counters")

    host = engine(spec, N, root, params, target, steps0)
    full = count_full_path(host)
    got = run(host, seq, overlapped=True)
    assert full[0] == 8, f"{full[0]} of {K} steps took the full path"
    assert_bits(ref, got, "host step index vs device claim")
    assert_bits(chain_counters(ser), chain_counters(host), "host step index vs device claim: chain counters")
    assert host._chain_T == K and bool((host.tile_sync == K).all())


@pytest.mark.gpu
def test_fast_path_follows_physics_steps_and_disturbance():
    """a call with physics_steps or a disturbance takes the full path, and the next plain call launches with what it left in cfg /
    buf (physics_steps kept, disturbance pointer cleared) -- the same bits as an engine stepped through the full path every time"""
    N = 4097
    spec, root, params, target, steps0, acts = inputs(N, "quiet")
    a, b = engine(spec, N, root, params, target, steps0), engine(spec, N, root, params, target, steps0)
    b._plain = False  # b's every call takes the full path
    dist = torch.rand(N, 6, generator=torch.Generator().manual_seed(3)).to(DEV) * 0.1
    calls = [dict(), dict(physics_steps=3), dict(), dict(disturbance=dist), dict(), dict(physics_steps=1), dict()]
    for i, kw in enumerate(calls * 2):
        for e in (a, b):
            e.position_task_step(acts[i % 4], **kw)
            if e is b:
                b._plain = False
    torch.cuda.synchronize()
    for k in ("root_state", "motor_thrust", "obs", "reward", "sim_steps"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert a._chain_T == b._chain_T == 2 * len(calls) and bool((a.tile_sync == a._chain_T).all())
    a.check(); b.check()


def test_reserved_step_index_is_refused():
    """by the C entry, called directly and through the _hostcall extension Hp1Engine uses; the extension checks its arguments"""
    from aerial_gym_simulator_b200 import hp1
    lib = _lib.load()
    assert lib.agx_hp1_position_task_step_at(None, None, None, 0xFFFFFFFF) == -1
    assert b"reserved" in lib.agx_last_error()
    entry = C.cast(lib.agx_hp1_position_task_step_at, C.c_void_p).value
    assert hp1._step_at(entry, 0, 0, 0, 0xFFFFFFFF) == -1
    assert b"reserved" in lib.agx_last_error()
    with pytest.raises(TypeError):
        hp1._step_at(entry, 0, 0, 0)
    with pytest.raises(ValueError):
        hp1._step_at(entry, 0, 0, 0, 1 << 32)
    with pytest.raises(ValueError):
        hp1._step_at(0, 0, 0, 0, 0)
