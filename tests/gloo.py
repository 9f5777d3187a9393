"""Multi-rank CPU checks: `run_ranks(fn, world, *args)` runs fn(rank, *args) on `world` spawned processes joined in one gloo
process group and returns what each rank returned, in rank order.

The ranks meet through a file store in a fresh temporary directory, so concurrent runs never share a rendezvous.  A rank
that raises sends its traceback and the call fails at once with it; on that, on a rank that dies, or on a timeout every rank
still running (typically blocked in a collective that waits for the failed one) is terminated, so no process outlives the
call."""
import os
import queue
import tempfile
import time
import traceback

import torch.distributed as dist
import torch.multiprocessing as mp


def _rank_main(fn, rank, world, store, args, results, received):
    try:
        dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
        out = fn(rank, *args)
    except BaseException:
        results.put((rank, traceback.format_exc(), None))
        return
    results.put((rank, None, out))
    # tensors travel as shared-memory file descriptors that the parent fetches from this process while it unpickles them:
    # stay alive until it has every result
    received.wait()
    dist.destroy_process_group()


def run_ranks(fn, world, *args, timeout=300):
    """fn must be a module-level function (the ranks import it by name) and its results must pickle."""
    ctx = mp.get_context("spawn")
    results, received = ctx.Queue(), ctx.Event()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_rank_main, args=(fn, r, world, os.path.join(tmp, "store"), args, results, received))
                 for r in range(world)]
        for p in procs:
            p.start()
        try:
            got, deadline = {}, time.monotonic() + timeout
            while len(got) < world:
                try:
                    rank, error, value = results.get(timeout=1.0)
                except queue.Empty:
                    for r, p in enumerate(procs):
                        if p.exitcode not in (None, 0):
                            raise RuntimeError(f"gloo rank {r} of {world} died with exit code {p.exitcode}") from None
                    if time.monotonic() > deadline:
                        raise RuntimeError(f"gloo ranks {sorted(set(range(world)) - set(got))} of {world} gave no result "
                                           f"within {timeout} s") from None
                    continue
                if error is not None:
                    raise RuntimeError(f"gloo rank {rank} of {world} failed:\n{error}")
                got[rank] = value
            received.set()
            for p in procs:
                p.join(timeout=60)
                assert p.exitcode == 0, (p.name, p.exitcode)
        finally:
            for p in procs:
                if p.is_alive():
                    p.terminate()
                p.join()
    return [got[r] for r in range(world)]
