"""Reasoning step bookkeeping fixtures: the reference's own code on the CPU over gloo, at data-parallel sizes 2 and 4:
    python tests/golden/make_golden_reasoning_step.py  ->  tests/golden/golden_reasoning_step.npz

Executed as the reference wrote them (extracted from its source with `ast` and compiled in place; only numerical
outputs are stored):
  - compute_rollout_metrics and compute_rollout_metrics_dynamic (rlinf/utils/distributed.py);
  - the tails of MegatronActor's and MegatronCritic's loss_func, from the early-stop all-reduce (actor) or the
    final-loss update (critic) to the return;
  - MegatronWorker._process_fwd_bwd_outputs for a training step over three micro-batches.
The functions see a `torch` whose CUDA device is the CPU and whose AVG all-reduce, which gloo lacks, is a SUM followed by
a division by the group size.  Megatron's average_losses_across_data_parallel_group is written from its documented
behaviour: concatenate, SUM all-reduce over data parallel, divide by the data-parallel size.  parallel_state's
data-parallel group is the world.

Cases (per rank r of P): unequal bsz; values present and absent; a multi-turn batch with uneven turns per
trajectory; an all-masked rank, which makes the reference raise; actor tails with early stop triggered on micro-batch 1
only, with the valid-token scale on and off; critic tails whose explained variance has count < 2, a zero centred
returns sum and a regular value."""
from __future__ import annotations

import ast
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden_response_rows import extract  # noqa: E402

L = 24
ACTOR_POLICY_KEYS = ("actor/policy_loss", "actor/policy_loss_abs", "actor/ratio", "actor/ratio_abs",
                     "actor/clipped_ratio", "actor/dual_cliped_ratio", "actor/approx_kl", "actor/clip_fraction")
ACTOR_KEYS = ACTOR_POLICY_KEYS + ("actor/final_loss", "actor/entropy_loss", "actor/kl_loss")
EV = tuple(f"__sum__/_critic_explained_variance/{k}"
           for k in ("count", "returns_sum", "returns_sq_sum", "errors_sum", "errors_sq_sum"))
CRITIC_KEYS = ("critic/value_loss", "critic/value_clip_ratio") + EV + ("critic/final_value_loss",)
N_MB = 3
EARLY_STOP = 1.5
ROLLOUT_CASES = ("values", "novalues", "dynamic", "empty")
ACTOR_CASES = {"vts": True, "novts": False}
CRITIC_CASES = ("regular", "count1", "flat")


def _torch_proxy():
    """torch with the CUDA device (by name or index) mapped to the CPU and ReduceOp.AVG done as SUM / size (gloo has no AVG)."""
    real_dist = torch.distributed

    def all_reduce(t, op=real_dist.ReduceOp.SUM, group=None, **kw):
        if op == real_dist.ReduceOp.AVG:
            real_dist.all_reduce(t, op=real_dist.ReduceOp.SUM, group=group)
            t.div_(real_dist.get_world_size(group))
            return None
        return real_dist.all_reduce(t, op=op, group=group, **kw)

    d = types.SimpleNamespace(**{k: getattr(real_dist, k) for k in dir(real_dist) if not k.startswith("__")})
    d.all_reduce = all_reduce
    cuda = types.SimpleNamespace(current_device=lambda: 0)

    class Proxy(types.ModuleType):
        def __getattr__(self, name):
            return getattr(torch, name)

    p = Proxy("torch")
    p.distributed = d
    p.cuda = cuda
    p.device = lambda s: torch.device("cpu")
    p.as_tensor = lambda data, dtype=None, device=None: torch.as_tensor(data, dtype=dtype)
    return p


def rollout_batch(case, rank):
    """Unequal bsz per rank; prompts of 3-9 tokens, responses of 0-L tokens at the end of the row."""
    g = torch.Generator().manual_seed(100 + 7 * rank + 31 * ROLLOUT_CASES.index(case))
    bsz = 3 + 2 * rank + (rank % 2)
    plen = torch.randint(3, 10, (bsz,), generator=g)
    rlen = torch.randint(0, L + 1, (bsz,), generator=g)
    rlen[0] = L
    S = 12 + L
    rmask = torch.zeros(bsz, S, dtype=torch.bool)
    for b in range(bsz):
        rmask[b, 12:12 + int(rlen[b])] = True
    if case == "empty" and rank == 1:
        rmask[:] = False
    batch = {"advantages": torch.randn(bsz, L, generator=g) * 1.7,
             "response_mask": rmask, "prompt_lengths": plen, "response_lengths": rlen,
             "rewards": torch.randn(bsz, generator=g), "is_end": torch.rand(bsz, generator=g) < 0.6}
    if case == "values":
        batch["values"] = torch.randn(bsz, L, generator=g) * 0.4 + 0.1
    if case == "dynamic":
        batch["response_mask"] = rmask[:, -L:].clone()
        turns, t = [], 0
        while len(turns) < bsz:  # 1, 2, 3 turns per trajectory, cut at bsz
            turns += [t] * (1 + t % 3)
            t += 1
        batch["idx_to_traj"] = turns[:bsz]
    return batch


def actor_inputs(rank, mb, P):
    g = torch.Generator().manual_seed(1000 + 17 * rank + 5 * mb + 101 * P)
    vals = (torch.rand(len(ACTOR_KEYS), generator=g) * 0.8 + 0.1)
    vals[ACTOR_KEYS.index("actor/ratio")] = 1.9 if mb == 1 else 0.9 + 0.2 * float(torch.rand(1, generator=g))
    loss = torch.randn((), generator=g) * 0.7
    bsz = 2 + rank
    mask = torch.rand(bsz, L, generator=g) < 0.7
    return vals, loss, mask


def critic_inputs(rank, mb, case, P):
    g = torch.Generator().manual_seed(5000 + 17 * rank + 5 * mb + 101 * P + 1009 * CRITIC_CASES.index(case))
    vals = torch.rand(len(CRITIC_KEYS), generator=g) * 0.8 + 0.1
    cnt = float(torch.randint(3, 40, (1,), generator=g))
    rs, es = float(torch.randn(1, generator=g)) * cnt * 0.3, float(torch.randn(1, generator=g)) * cnt * 0.2
    ev = [cnt, rs, rs * rs / cnt + cnt * 0.5, es, es * es / cnt + cnt * 0.3]
    if case == "count1":
        ev = [0.0, 0.0, 0.0, 0.0, 0.0] if (rank, mb) != (0, 0) else [1.0, 0.5, 0.25, 0.1, 0.01]
    if case == "flat":
        ev = [2.0, 2.0, 2.0, 0.5, 0.3]  # every return is 1: returns_sq_sum - returns_sum^2 / count == 0
    vals[2:7] = torch.tensor(ev)
    loss = torch.randn((), generator=g) * 0.5
    return vals, loss


def _tail(path, class_name, first, globs):
    """loss_func's statements from the one `first` selects to the return, compiled as
    tail(self, loss, metrics_data, mask, entropy_loss, kl_loss) -> (loss, metrics_data)."""
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == class_name)
    fn = next(n for n in ast.walk(cls) if isinstance(n, ast.FunctionDef) and n.name == "loss_func")
    start = next(i for i, st in enumerate(fn.body) if first(st))
    args = ast.arguments(posonlyargs=[], args=[ast.arg(arg=a) for a in ("self", "loss", "metrics_data", "mask",
                                                                         "entropy_loss", "kl_loss")],
                         kwonlyargs=[], kw_defaults=[], defaults=[])
    tail = ast.FunctionDef(name="tail", args=args, body=fn.body[start:], decorator_list=[], returns=None,
                           type_params=[])
    mod = ast.Module(body=[tail], type_ignores=[])
    ast.fix_missing_locations(mod)
    exec(compile(mod, path, "exec"), globs)
    return globs["tail"]


def _worker(rank, P, init_file, out_dir):
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=P)
    ref = ref_loader.load_reference()
    root = ref_loader.REFERENCE_ROOT
    tp = _torch_proxy()
    mu = ref.metric_utils

    def average_losses_across_data_parallel_group(losses):
        averaged = torch.cat([x.clone().detach().view(1) for x in losses])
        dist.all_reduce(averaged, group=None)
        return averaged / dist.get_world_size()

    pstate = types.SimpleNamespace(get_data_parallel_group=lambda: None,
                                   get_data_parallel_world_size=lambda: dist.get_world_size())
    globs = {"torch": tp, "Worker": sys.modules["rlinf.scheduler"].Worker, "Optional": __import__("typing").Optional,
             "ProcessGroup": object, "parallel_state": pstate,
             "average_losses_across_data_parallel_group": average_losses_across_data_parallel_group,
             "CRITIC_EXPLAINED_VARIANCE_STAT_KEYS": mu.CRITIC_EXPLAINED_VARIANCE_STAT_KEYS,
             "CRITIC_EXPLAINED_VARIANCE_KEY": mu.CRITIC_EXPLAINED_VARIANCE_KEY,
             "compute_critic_explained_variance_from_stats": mu.compute_critic_explained_variance_from_stats,
             "get_last_rank": lambda: dist.get_world_size() - 1,
             "broadcast_tensor_within_pp": lambda x: x}
    fns = extract(os.path.join(root, "rlinf/utils/distributed.py"),
                  ["compute_rollout_metrics", "compute_rollout_metrics_dynamic"], globs)
    actor_tail = _tail(os.path.join(root, "rlinf/workers/actor/megatron_actor_worker.py"), "MegatronActor",
                       lambda st: isinstance(st, ast.AnnAssign) and getattr(st.target, "id", "") == "_imp", globs)
    critic_tail = _tail(os.path.join(root, "rlinf/workers/critic/megatron_critic_worker.py"), "MegatronCritic",
                        lambda st: "metrics_data.update" in ast.unparse(st), globs)
    process = extract(os.path.join(root, "rlinf/workers/megatron_worker.py"), ["_process_fwd_bwd_outputs"], globs,
                      class_name="MegatronWorker")["_process_fwd_bwd_outputs"]

    res = {}
    for case in ROLLOUT_CASES:
        b = rollout_batch(case, rank)
        fn = fns["compute_rollout_metrics_dynamic" if case == "dynamic" else "compute_rollout_metrics"]
        try:
            m, tpl, tdl = fn(b, 12, L, data_parallel_group=None)
            res[f"rollout_{case}_keys"] = np.array(list(m.keys()))
            res[f"rollout_{case}_vals"] = np.array([float(v) for v in m.values()], dtype=np.float64)
            res[f"rollout_{case}_plens"] = tpl.numpy()
            res[f"rollout_{case}_dlens"] = tdl.numpy()
        except Exception as e:  # noqa: BLE001 - the all-masked rank: the reference's error is the datum
            res[f"rollout_{case}_error"] = np.array(type(e).__name__)
            # the other ranks wait in the advantages' MAX all-reduce: take part in it so that they finish
            dist.all_reduce(torch.zeros(2), op=dist.ReduceOp.MAX)

    for case, vts in ACTOR_CASES.items():
        outs = []
        gvt_total = sum(float(actor_inputs(r, mb, P)[2].sum()) for r in range(P) for mb in range(N_MB))
        for mb in range(N_MB):
            vals, loss, mask = actor_inputs(rank, mb, P)
            md = {k: vals[i].clone() for i, k in enumerate(ACTOR_POLICY_KEYS)}
            self = types.SimpleNamespace(
                cfg=types.SimpleNamespace(algorithm=types.SimpleNamespace(early_stop_imp_ratio=EARLY_STOP,
                                                                          use_valid_token_scale=vts)),
                global_valid_token=torch.tensor(gvt_total, dtype=torch.float32) / N_MB, num_microbatches=N_MB,
                log_warning=lambda msg: None)
            out_loss, md = actor_tail(self, loss.clone(), md, mask,
                                      vals[ACTOR_KEYS.index("actor/entropy_loss")].clone(),
                                      vals[ACTOR_KEYS.index("actor/kl_loss")].clone())
            res[f"actor_{case}_mb{mb}_loss"] = out_loss.detach().numpy()
            res[f"actor_{case}_mb{mb}_metrics"] = np.array([float(md[k]) for k in ACTOR_KEYS], dtype=np.float32)
            outs.append(md)
        step = process(types.SimpleNamespace(enable_dynamic_batch_size=False), outs, False)
        res[f"actor_{case}_step_keys"] = np.array(list(step.keys()))
        res[f"actor_{case}_step_vals"] = np.array(list(step.values()), dtype=np.float64)

    for case in CRITIC_CASES:
        outs = []
        for mb in range(N_MB):
            vals, loss = critic_inputs(rank, mb, case, P)
            md = {k: vals[i].clone() for i, k in enumerate(CRITIC_KEYS) if k != "critic/final_value_loss"}
            out_loss, md = critic_tail(None, loss.clone(), md, None, None, None)
            res[f"critic_{case}_mb{mb}_loss"] = out_loss.detach().numpy()
            res[f"critic_{case}_mb{mb}_metrics"] = np.array([float(md[k]) for k in CRITIC_KEYS], dtype=np.float32)
            outs.append(md)
        step = process(types.SimpleNamespace(enable_dynamic_batch_size=False), outs, False)
        res[f"critic_{case}_step_keys"] = np.array(list(step.keys()))
        res[f"critic_{case}_step_vals"] = np.array(list(step.values()), dtype=np.float64)
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), **res)
    dist.destroy_process_group()


def main():
    out = {"L": np.array(L), "n_mb": np.array(N_MB), "early_stop": np.array(EARLY_STOP)}
    for P in (2, 4):
        with tempfile.TemporaryDirectory() as tmp:
            mp.spawn(_worker, args=(P, os.path.join(tmp, "init"), tmp), nprocs=P, join=True)
            for r in range(P):
                for k, v in np.load(os.path.join(tmp, f"r{r}.npz")).items():
                    out[f"P{P}_r{r}_{k}"] = v
    path = os.path.join(HERE, "golden_reasoning_step.npz")
    np.savez_compressed(path, **out)
    print(path, len(out))


if __name__ == "__main__":
    main()
