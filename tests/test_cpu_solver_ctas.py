"""CPU: how many CTAs stay with the inertial solve while the others work the deferred weights queue (solver_plan.py's
model of chain_solver_ctas in vc_engine.inl).  The rule keeps the most solver CTAs for which the CTAs that leave by the
end of elimination level 1 take every 16-interval weight task in one round; where no count does, it falls back to
`chain_plan.n_solver`.  Assumes an H100 SXM: 132 SMs."""
import pytest

import chain_plan as cp
import solver_plan as sp

FRAMES = sorted({n for n, _ in cp.chain_cases()} | {2000, 5000, 10000})


def test_target_takes_one_round():
    """2000 frames: 125 tasks; with 7 solver CTAs, 7 CTAs leave at the start (250 chunks for 264 groups: CTAs 125..131
    have none), 93 after level 0 and 25 after level 1 (32 chunks, then 7 go on)."""
    assert cp.level_sizes(2000) == [2000, 250, 32, 4] and cp.weight_tasks(2000) == 125
    assert sp.solver_ctas(2000) == 7 and sp.weight_rounds(2000) == 1
    assert sp.early_leavers(2000, 7) == 125 and sp.early_leavers(2000, 8) == 124


@pytest.mark.parametrize("n_frames", FRAMES)
def test_one_round_wherever_the_rule_applies(n_frames):
    tasks = cp.weight_tasks(n_frames)
    ns = sp.solver_ctas(n_frames)
    if sp.one_round_possible(n_frames):
        assert 1 <= ns < cp.H100_SMS
        assert sp.early_leavers(n_frames, ns) >= tasks
        assert ns == cp.H100_SMS - 1 or sp.early_leavers(n_frames, ns + 1) < tasks  # the most that do
        assert sp.weight_rounds(n_frames) == 1
    else:
        assert ns == cp.n_solver(n_frames)


def test_rule_and_fallback_boundaries():
    """Up to 2000 frames every rig takes its tasks in one round; from 2049 frames (a fifth level: at least 5 CTAs stay
    after level 1, and 128 tasks) the rule falls back to 8 solver CTAs."""
    assert all(sp.weight_rounds(n) == 1 for n in range(2, 2001))
    assert not sp.one_round_possible(2049)
    assert sp.solver_ctas(2049) == 8 and sp.weight_rounds(2049) == 2
    assert sp.solver_ctas(5000) == 8 and sp.weight_rounds(5000) == 3
    assert sp.solver_ctas(10000) == 8 and sp.weight_rounds(10000) == 6
    assert sp.solver_ctas(5) == 131 and sp.solver_ctas(1056) == 66
