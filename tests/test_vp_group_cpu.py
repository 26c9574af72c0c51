"""Which process group the vocabulary-parallel ops split the vocabulary over when none is passed, on a 2-rank gloo world
on the CPU: Megatron's tensor-parallel group when its model parallelism is initialised, and an error, before any device
work, when it is not (the world group of a data-parallel job is not the tensor-parallel group)."""
import os
import socket
import sys
import types

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rlinf_b200 import ops

        logits = torch.zeros(2, 3, 10)
        target = torch.zeros(2, 3, dtype=torch.int64)
        hidden = torch.zeros(6, 64, dtype=torch.bfloat16)
        weight = torch.zeros(10, 64, dtype=torch.bfloat16)
        calls = [lambda: ops.vocab_parallel_entropy_and_log_probs(logits, target),
                 lambda: ops.vocab_parallel_log_probs_from_logits(logits, target),
                 lambda: ops.vocab_parallel_linear_logprobs_entropy(hidden, weight, target)]
        for call in calls:
            try:
                call()
                raise AssertionError("a 2-rank world without a group must be rejected")
            except ValueError as e:
                assert "group=" in str(e), str(e)
        # an explicit group is used as given
        assert ops._vp_group(dist.group.WORLD, "t")[1:] == (world, rank)
        # Megatron's tensor-parallel group, when its model parallelism is initialised (one rank per group here)
        singles = [dist.new_group([r]) for r in range(world)]
        ps = types.ModuleType("megatron.core.parallel_state")
        ps.model_parallel_is_initialized = lambda: True
        ps.get_tensor_model_parallel_group = lambda: singles[rank]
        core = types.ModuleType("megatron.core")
        core.parallel_state = ps
        sys.modules.update({"megatron": types.ModuleType("megatron"), "megatron.core": core,
                            "megatron.core.parallel_state": ps})
        group, P, k = ops._vp_group(None, "t")
        assert group is singles[rank] and (P, k) == (1, 0)
        ps.model_parallel_is_initialized = lambda: False
        try:
            ops._vp_group(None, "t")
            raise AssertionError("uninitialised Megatron model parallelism must not resolve to the world")
        except ValueError:
            pass
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_group_none_resolves_to_megatron_tp_group_or_is_rejected():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert res == {0: "ok", 1: "ok"}, res
