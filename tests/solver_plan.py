"""Host model of how many CTAs stay with the inertial chain solve while the others work the deferred weights queue:
`chain_solver_ctas` (vc_engine.inl), in plain Python, on top of the level table of chain_plan.py.

The host keeps the most solver CTAs, at least 1, for which the CTAs that leave at the start, after elimination level 0
or after level 1 take every 16-interval weight task in one round.  Where no count does that (more tasks than CTAs can
leave by then), it falls back to `chain_plan.n_solver`: between 8 and 32.
"""
import math

import chain_plan as cp


def early_leavers(n_frames, ns, sms=cp.H100_SMS, narrow_ok=True):
    """CTAs that leave the solve at the start, after level 0 or after level 1 with ns solver CTAs: the kernel's rule for
    who goes on after a level (everybody the next level needs, never fewer than ns); with nothing to eliminate all but
    ns leave at the barrier before the Schur reduction."""
    sizes = cp.level_sizes(n_frames)
    nl = len(sizes)
    if nl == 1:
        return sms - ns
    n_act = sms
    for l in range(min(nl - 1, 2)):
        n_next = ns
        if l + 2 < nl:
            nsep2 = sizes[l + 2]
            n_next = sms if (nsep2 > sms or not narrow_ok) else max(ns, nsep2)
        n_act = min(n_next, n_act)
    return sms - n_act


def one_round_possible(n_frames, sms=cp.H100_SMS, narrow_ok=True):
    return any(early_leavers(n_frames, k, sms, narrow_ok) >= cp.weight_tasks(n_frames) for k in range(1, sms))


def solver_ctas(n_frames, sms=cp.H100_SMS, narrow_ok=True):
    """CTAs that stay with the solve while the others work the weights queue (ChainSolveArgs::n_solver)."""
    tasks = cp.weight_tasks(n_frames)
    for ns in range(sms - 1, 0, -1):
        if early_leavers(n_frames, ns, sms, narrow_ok) >= tasks:
            return ns
    return cp.n_solver(n_frames, sms)


def weight_rounds(n_frames, sms=cp.H100_SMS):
    """Rounds of the weights queue: tasks per CTA that leaves the solve, rounded up."""
    return math.ceil(cp.weight_tasks(n_frames) / (sms - min(solver_ctas(n_frames, sms), sms)))
