"""CPU checks of in-flight batching's host loop (vlm-fo1_b200/pipeline.py: refill_need, run_slots) against a fake slot pool that
decodes one token per running slot per step: the admission policy, that every request completes exactly once, completion order,
and refused admissions."""
from importlib import import_module

import pytest


def _P():
    return import_module("vlm-fo1_b200.pipeline")


class FakePool:
    """Request i runs lengths[i] steps after its admission (column 0 is recorded at admission: a length-1 request finishes there)."""

    def __init__(self, n_slots, lengths, refuse=()):
        self.n, self.lengths, self.refuse = n_slots, lengths, set(refuse)
        self.left = [0] * n_slots
        self.item = [None] * n_slots
        self.log = []          # ("admit", items, slots, free before) / ("decode", exit_at, running before, steps)

    def admit(self, items, slots):
        free = sum(1 for b in range(self.n) if self.left[b] == 0 and self.item[b] is None)
        self.log.append(("admit", list(items), list(slots), free))
        done = []
        for it, b in zip(items, slots):
            assert self.item[b] is None, "slot admitted twice"
            if it in self.refuse:
                continue
            self.item[b], self.left[b] = it, self.lengths[it] - 1
            done.append(it)
        return done

    def running(self):
        return sum(1 for b in range(self.n) if self.item[b] is not None and self.left[b] > 0)

    def decode(self, exit_at):
        steps, before = 0, self.running()
        while self.running() > exit_at:
            for b in range(self.n):
                if self.item[b] is not None and self.left[b] > 0:
                    self.left[b] -= 1
            steps += 1
        self.log.append(("decode", exit_at, before, steps))
        return steps

    def poll(self):
        fin = [int(self.item[b] is None or self.left[b] == 0) for b in range(self.n)]
        lens = [self.lengths[self.item[b]] if self.item[b] is not None else 0 for b in range(self.n)]
        return fin, lens

    def take(self, slot):
        it, self.item[slot] = self.item[slot], None
        return it


def _run(n_slots, lengths, refuse=()):
    P = _P()
    pool = FakePool(n_slots, lengths, refuse)
    out = []
    for it, b, n in P.run_slots(len(lengths), n_slots, pool.admit, pool.decode, pool.poll):
        assert pool.take(b) == it and n == lengths[it]
        out.append(it)
    return pool, out


def test_refill_need():
    P = _P()
    assert P.refill_need(16, 100) == 4 and P.refill_need(16, 2) == 2 and P.refill_need(16, 0) == 0
    assert P.refill_need(3, 100) == 1 and P.refill_need(1, 5) == 1 and P.refill_need(32, 9) == 8


@pytest.mark.parametrize("n_slots", [1, 3, 4, 8])
def test_every_request_completes_once(n_slots):
    lengths = [1 + (7 * i * i + 3 * i) % 23 for i in range(29)]
    pool, out = _run(n_slots, lengths)
    assert sorted(out) == list(range(len(lengths)))
    admitted = [it for e in pool.log if e[0] == "admit" for it in e[1]]
    assert admitted == list(range(len(lengths)))                  # queue order


def test_admission_policy():
    n_slots = 8
    lengths = [3 + (5 * i) % 17 for i in range(40)]
    pool, _ = _run(n_slots, lengths)
    queued = len(lengths)
    for e in pool.log:
        if e[0] == "admit":
            _, items, slots, free = e
            # a refill waits for a quarter of the pool, or for room for the whole (shorter) queue; then it fills every free slot
            assert free >= min(2, queued) and len(items) == min(free, queued)
            assert slots == sorted(slots)
            queued -= len(items)
        else:
            _, exit_at, before, _ = e
            assert exit_at == (n_slots - min(2, queued) if queued else 0)
    assert queued == 0


def test_completion_order():
    lengths = [30, 2, 9, 2, 1, 15, 4, 4]
    _, out = _run(2, lengths)
    # slot 0 runs request 0 (29 steps after its column 0); slot 1 works through the rest in queue order (request 4 finishes at its
    # admission); requests 0 and 7 end in the last segment, which reports them in slot order
    assert out == [1, 2, 3, 4, 5, 6, 0, 7]


def test_refused_admission_frees_its_slot():
    lengths = [4, 5, 6, 2, 3, 7]
    pool, out = _run(3, lengths, refuse={1, 4})
    assert sorted(out) == [0, 2, 3, 5]
    assert all(pool.item[b] is None for b in range(3))
