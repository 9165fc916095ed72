"""CPU model of the unit-queue ticket protocol (robosuite_b200/csrc/b2s_unit.cuh): an event-driven simulation of B lockstep blocks that take
tickets from the ring, run one round (all of a block's units finish together: stage barriers) and publish the environments for their next
substep.  It pins the property the kernel relies on: every control step terminates with every unit executed exactly once."""
import heapq

import numpy as np
import pytest


def simulate(n_env, nsub, n_blocks, wpb, policy, seed=0, max_events=10 ** 6):
    """policy 'produced': a block takes min(wpb, tail - head) tickets that already exist (the shipped kernel);
    'eager': a block takes wpb tickets whether produced or not and starts its round only when ALL of them have arrived (stage barrier in
    front of the first stage).  Returns (finished units, deadlocked?)."""
    rng = np.random.default_rng(seed)
    total = n_env * nsub
    ring = [-1] * total
    for e in range(n_env):
        ring[e] = e  # env + n_env * substep
    head, tail, done = 0, n_env, 0
    executed = np.zeros(total, dtype=np.int64)
    now = 0.0
    events = []  # (time, block): the block's round finishes
    waiting = {}  # block -> tickets it holds while some are missing (eager) / [] when it found no ticket (produced)
    idle = list(range(n_blocks))

    def try_start(b):
        nonlocal head
        if policy == "produced":
            if head >= total:
                return True  # exits
            k = min(wpb, tail - head)
            if k <= 0:
                waiting[b] = []
                return False
            mine = list(range(head, head + k)); head += k
        else:
            mine = waiting.pop(b, None)
            if mine is None:
                if head >= total:
                    return True
                mine = list(range(head, min(head + wpb, total))); head += len(mine)
            if any(ring[t] < 0 for t in mine):
                waiting[b] = mine
                return False
        dur = 1.0 + rng.exponential(0.5)
        heapq.heappush(events, (now + dur, b, tuple(mine)))
        return False

    for b in list(idle):
        try_start(b)
    n_ev = 0
    while events and n_ev < max_events:
        n_ev += 1
        now, b, mine = heapq.heappop(events)
        for t in mine:
            code = ring[t]
            env, sub = code % n_env, code // n_env
            executed[sub * n_env + env] += 1
            if sub + 1 < nsub:
                ring[tail] = env + n_env * (sub + 1); tail += 1
            done += 1
        try_start(b)
        for w in list(waiting):  # blocks that were waiting look again
            if policy == "produced":
                waiting.pop(w)
            try_start(w)
    deadlock = done < total
    return done, deadlock, executed


@pytest.mark.parametrize("n_env,n_blocks,wpb", [(16, 2, 8), (64, 8, 8), (64, 4, 16), (200, 9, 16), (4096, 146, 16)])
def test_taking_only_produced_tickets_always_terminates(n_env, n_blocks, wpb):
    nsub = 25 if n_env < 4096 else 5
    for seed in range(3):
        done, dead, executed = simulate(n_env, nsub, n_blocks, wpb, "produced", seed)
        assert not dead and done == n_env * nsub
        assert (executed == 1).all()  # every environment-substep exactly once


def test_eager_ticket_taking_terminates_in_the_model_too():
    """the first lockstep version took `wpb` tickets whether produced or not and waited for them in front of the first stage barrier.  On
    the GPU it stalled until the watchdog in every control step; in THIS model it terminates, i.e. the stall was
    not a property of the ticket arithmetic - the shipped kernel removes the wait altogether instead of relying on it"""
    for seed in range(3):
        done, dead, executed = simulate(64, 25, 8, 8, "eager", seed)
        assert not dead and (executed == 1).all()
