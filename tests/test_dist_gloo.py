"""N > 1 path on CPU: two gloo ranks, servers sharded round-robin, one all-gather of winners.
The local solver here is the CPU oracle (test stand-in for the per-rank GPU engine); the
sharding / packing / collective / reassembly code is the product's (parallel.py)."""
import os
import socket
import sys

import numpy as np
import torch.multiprocessing as mp
from tests.levels import limited_fleet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    import oracle
    from workload_variant_autoscaler_b200 import Allocs, parallel, synth_fleet
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fleet = synth_fleet(13, 3, seed=77, max_batch_choices=(2, 4, 8))

    def solve_local(shard):
        _, win = oracle.solve(shard)
        a = Allocs(shard.n_servers)
        for name in ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate"):
            getattr(a, name)[:] = win[name]
        return a

    full = parallel.solve_sharded(solve_local, fleet, rank=rank, world=world, all_gather=parallel.torch_all_gather())
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **full.columns())
    dist.barrier()
    dist.destroy_process_group()


def _limited_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    import oracle
    from workload_variant_autoscaler_b200 import Allocs, parallel
    from workload_variant_autoscaler_b200._abi import ALLOC_COLUMNS, SAT_PRIORITY_ROUND_ROBIN
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fleet = limited_fleet(19, 9, SAT_PRIORITY_ROUND_ROBIN, delayed=True, n=23)

    def analyze_local(shard):  # stand-in for Engine.analyze on this rank's GPU
        c = oracle.calculate(shard).reshape(-1)
        a = Allocs(c.size)
        for name, _ in ALLOC_COLUMNS:
            getattr(a, name)[:] = c[name]
        return a

    cand, win = parallel.solve_sharded_limited(analyze_local, fleet, rank=rank, world=world,
                                               all_gather=parallel.torch_all_gather())
    np.savez(os.path.join(out_dir, f"lim{rank}.npz"), **{"w_" + k: v for k, v in win.columns().items()},
             **{"c_" + k: v for k, v in cand.columns().items()})
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_limited_mode_matches_single_greedy(tmp_path, oracle_mod):
    """Limited mode at world_size 2: candidates generated per shard, one all-gather of the candidate tables, the
    product's SolveGreedy (host C++) run redundantly on both ranks; both equal the oracle's single-process greedy."""
    from workload_variant_autoscaler_b200._abi import SAT_PRIORITY_ROUND_ROBIN
    world = 2
    mp.spawn(_limited_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    fleet = limited_fleet(19, 9, SAT_PRIORITY_ROUND_ROBIN, delayed=True, n=23)
    cand_o, win_o = oracle_mod.solve(fleet)
    for r in range(world):
        got = np.load(os.path.join(tmp_path, f"lim{r}.npz"))
        for prefix, want_s in (("w_", win_o), ("c_", cand_o.reshape(-1))):
            for name in want_s.dtype.names:
                want = np.ascontiguousarray(want_s[name])
                g = got[prefix + name]
                if want.dtype == np.float32:
                    assert np.array_equal(g.view(np.uint32), want.view(np.uint32)), (r, prefix, name)
                else:
                    assert np.array_equal(g.astype(np.int64), want.astype(np.int64)), (r, prefix, name)


def test_sharded_unlimited_refuses_limited_fleet():
    from workload_variant_autoscaler_b200 import parallel
    import pytest
    with pytest.raises(ValueError):
        parallel.solve_sharded(lambda s: None, limited_fleet(3, 5), rank=0, world=2, all_gather=lambda b: b)


def test_two_rank_sharded_solve_matches_single(tmp_path, oracle_mod):
    from workload_variant_autoscaler_b200 import synth_fleet
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    fleet = synth_fleet(13, 3, seed=77, max_batch_choices=(2, 4, 8))
    _, win = oracle_mod.solve(fleet)
    for r in range(world):
        got = np.load(os.path.join(tmp_path, f"rank{r}.npz"))
        for name in win.dtype.names:
            want = np.ascontiguousarray(win[name])
            g = got[name]
            if want.dtype == np.float32:
                assert np.array_equal(g.view(np.uint32), want.view(np.uint32)), name
            else:
                assert np.array_equal(g.astype(np.int64), want.astype(np.int64)), name
