"""CPU tier: parallel.plan_token_batches, the serving plan for batches of mixed token counts (the style sampler runs on
packed token rows, so a batch may mix any token counts): every utterance once, the batch bounds, determinism, and rank
loads within one batch's cost of each other."""
import random

import pytest

from styletts2_b200.parallel import plan_token_batches


def _queue(n, seed):
    r = random.Random(seed)
    return [r.randint(16, 256) for _ in range(n)]


@pytest.mark.parametrize("n,world,max_batch,max_rows,seed", [(32, 1, 32, 8192, 0), (32, 2, 8, 1024, 1), (100, 3, 16, 2000, 2),
                                                             (7, 8, 4, 600, 3), (257, 4, 32, 4096, 4), (50, 2, 1, 256, 5)])
def test_plan_token_batches(n, world, max_batch, max_rows, seed):
    lengths = _queue(n, seed)
    plan = plan_token_batches(lengths, world, max_batch, max_rows)
    assert len(plan) == world
    flat = [i for rank in plan for batch in rank for i in batch]
    assert sorted(flat) == list(range(n))                                 # every index exactly once
    costs = []
    for rank in plan:
        for batch in rank:
            assert 1 <= len(batch) <= max_batch
            assert sum(lengths[i] for i in batch) <= max_rows
            costs.append(sum(lengths[i] for i in batch))
    loads = [sum(lengths[i] for batch in rank for i in batch) for rank in plan]
    assert max(loads) - min(loads) <= max(costs)
    assert plan == plan_token_batches(list(lengths), world, max_batch, max_rows)     # deterministic


def test_plan_token_batches_mixes_token_counts():
    """unlike plan_equal_length_batches, distinct token counts share a batch"""
    lengths = [16, 17, 200, 31, 64]
    plan = plan_token_batches(lengths, 1, 32, 10000)
    assert plan == [[[2, 4, 3, 1, 0]]]


def test_plan_token_batches_rejects_an_utterance_over_max_rows():
    with pytest.raises(ValueError):
        plan_token_batches([10, 300], 1, 4, 256)
