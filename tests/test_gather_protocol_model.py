"""The multi-GPU step loop's launch / residency protocol (DESIGN section 9) as an exhaustively explored model (tests/_protocol_model.py):
the three failures seen on hardware are reachable deadlocks of the earlier designs, and the shipped design (ring gate in front
of the step, one-warp ready gate in front of the push) has none -- under an adversarial CTA scheduler -- as long as the GPU holds one
step grid plus one ready gate per ring slot, whatever the number and the footprint of the push CTAs.  Abstract slots, no timing: the
hardware check is tests/test_multi_gpu.py."""
import itertools

import pytest

from tests._protocol_model import Protocol


def explore(**kw):
    p = Protocol(**kw)
    states, deadlocks, violations = p.explore()
    return p, states, deadlocks, violations


def test_unprotected_ring_is_unsafe():
    _, _, dead, bad = explore(steps=5, tiles=2, slots=4, ring=2, push_ctas=1, design="none")
    assert not dead and bad and "overwrote ring slot" in bad[0]


def test_lesson_1_in_kernel_back_pressure_deadlocks():
    """the first multi-GPU design: the tiles of step T+ring spin for push T while they and their chained successor
    hold every CTA slot, so the push never becomes resident.  Safe, but not live unless the GPU holds several whole step grids."""
    p, _, dead, bad = explore(steps=5, tiles=2, slots=4, ring=2, push_ctas=1, design="backpressure")
    assert not bad and dead
    assert any("step3:RESIDENT/RESIDENT, step4:RESIDENT/RESIDENT" in p.describe(d) for d in dead)
    # the gate kernel in front of the step: a step that is held back is not resident
    _, _, dead, bad = explore(steps=5, tiles=2, slots=4, ring=2, push_ctas=1, design="gate")
    assert not dead and not bad


def test_lesson_2_a_push_cta_with_a_large_footprint_starves_the_all_arrive_step():
    """carve-out poisoning: one push CTA on an idle SM cost the space of several step CTAs (24 push CTAs cost > 160 slots)"""
    kw = dict(steps=4, tiles=3, slots=6, ring=2, push_ctas=1, design="gate", rare={1})
    assert not explore(push_weight=1, **kw)[2]
    assert explore(push_weight=2, **kw)[2]


def test_lesson_3_spinning_pushes_are_not_free_even_when_they_fit_on_paper():
    """tiles + push_ctas <= slots, yet one push per ring slot may be resident and spinning for its producer when the step that needs its
    whole grid co-resident comes up (engine error word 3 + 'push of epoch 3 never saw its producer' at 2 and 4 GPUs)"""
    kw = dict(steps=5, tiles=3, slots=4, ring=2, push_ctas=1, design="gate")
    assert not explore(rare=(), **kw)[2]          # ordinary steps drain tile by tile
    p, _, dead, bad = explore(rare={2}, **kw)
    assert dead and not bad
    # the one-warp ready gate: the push CTAs are not resident while they would only wait -- but the gates themselves are, so the
    # reserve must cover one of them per ring slot
    assert explore(steps=5, tiles=3, slots=4, ring=2, push_ctas=1, design="final", rare={2})[2]
    assert not explore(steps=5, tiles=3, slots=5, ring=2, push_ctas=1, design="final", rare={2})[2]


@pytest.mark.parametrize("tiles,ring,push_ctas,push_weight", [c for c in itertools.product((2, 3), (2, 3), (1, 2, 3), (1, 2))
                                                               if c[2] * c[3] <= c[0] + c[1]])
def test_shipped_design_is_live_and_safe_with_a_reserve_of_one_slot_per_ring_slot(tiles, ring, push_ctas, push_weight):
    """every step rare (the worst case), adversarial scheduler: no deadlock and no overwrite with slots = tiles + ring, for every push
    shape that fits the GPU by itself; and the bound is tight (csrc/hp1.cu: kCoopReserve = 32 slots against a ring of 4)"""
    steps = 2 * ring + 1
    rare = set(range(1, steps + 1))
    _, states, dead, bad = explore(steps=steps, tiles=tiles, slots=tiles + ring, ring=ring, push_ctas=push_ctas, push_weight=push_weight,
                                   design="final", rare=rare)
    assert states > 100 and not dead and not bad
    _, _, dead, _ = explore(steps=steps, tiles=tiles, slots=tiles + ring - 1, ring=ring, push_ctas=push_ctas, push_weight=push_weight,
                            design="final", rare=rare)
    assert dead
