import multiprocessing
import time

import pytest
import torch.distributed as dist

from tests.gloo import run_ranks


def _rank_1_raises(rank):
    if rank == 1:
        raise ValueError("rank 1 gives up")
    dist.barrier()  # rank 0 waits here for a rank that never comes


def test_a_failing_rank_fails_the_call_at_once_and_leaves_no_process():
    t0 = time.monotonic()
    with pytest.raises(RuntimeError, match="(?s)rank 1 of 2 failed.*ValueError: rank 1 gives up"):
        run_ranks(_rank_1_raises, 2, timeout=600)
    assert time.monotonic() - t0 < 60  # process start-up only, not the timeout
    assert multiprocessing.active_children() == []
