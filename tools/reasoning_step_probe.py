"""Times the reasoning step bookkeeping on one GPU against the reference's eager chain restated in plain torch:

  - epilogue: MegatronLossEpilogue per micro-batch (actor, early stop and valid-token scale on, 11 keys) against the
    reference's loss_func tail (clone of actor/ratio, the early-stop test read on the host, mask.sum() / gvt * dp *
    num_microbatches read with .item(), one concatenate-and-divide per key);
  - step: step_metrics over 8 micro-batches against _process_fwd_bwd_outputs (a stack, a mean and a .cpu().item() per
    key);
  - rollout: compute_rollout_metrics (values present) at bsz 512 x L 8,192 against the reference's
    compute_rollout_metrics restated (the sums read one by one with .item(), masked_select, min / max, the length
    statistics on the host).
Data-parallel peers are emulated: collectives are counted, not made, so the times are the device and host work alone.
Reports the times, host syncs and collectives per call, and the card name and power limit read in the same run;
prints one JSON line, also written to --out if given.

    python tools/reasoning_step_probe.py [--reps 5] [--iters 20] [--out result.json]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from rlinf_b200.algorithms import MegatronLossEpilogue, step_metrics  # noqa: E402
from rlinf_b200.utils import distributed as RD  # noqa: E402
from reasoning_loss_probe import card, host_syncs, timed  # noqa: E402

KEYS = ("actor/policy_loss", "actor/policy_loss_abs", "actor/ratio", "actor/ratio_abs", "actor/clipped_ratio",
        "actor/dual_cliped_ratio", "actor/approx_kl", "actor/clip_fraction", "actor/final_loss", "actor/entropy_loss",
        "actor/kl_loss")
N_MB = 8


class Counter:
    """torch.distributed stand-in of a 2-rank data-parallel group whose peers hold this rank's buffers."""

    def __init__(self):
        self.n = 0

    def is_available(self):
        return True

    def is_initialized(self):
        return True

    def get_world_size(self, group=None):
        return 2

    def all_reduce(self, t, op=None, group=None):
        self.n += 1
        t.mul_(2)

    def all_gather_into_tensor(self, out, inp, group=None):
        self.n += 1
        out.copy_(torch.stack([inp, inp]).reshape(out.shape))


def epilogue_inputs():
    g = torch.Generator(device="cuda").manual_seed(0)
    metrics = {k: torch.rand((), device="cuda", generator=g) for k in KEYS}
    loss = torch.randn((), device="cuda", generator=g)
    mask = torch.rand(64, 2048, device="cuda", generator=g) < 0.7
    gvt = (mask.sum() * 2 * N_MB).float().reshape(1)
    return metrics, loss, mask, gvt


def ref_tail(metrics, loss, mask, gvt, dp=2):
    imp = metrics["actor/ratio"].clone()
    dist.all_reduce(imp)
    imp = imp / dp
    if imp > 10.0:
        loss = loss * 0.0
    scale = mask.sum() / gvt * dp * N_MB
    loss = loss * scale.item()
    out = {}
    for k, v in metrics.items():
        avg = torch.cat([v.clone().detach().view(1)])
        dist.all_reduce(avg)
        out[k] = avg / dp
    out["actor/final_loss"] = loss.detach()
    return loss, out


def ref_step(outs):
    res = {}
    for k in outs[0]:
        res[k] = torch.stack([o[k] for o in outs]).mean().cpu().item()
    return res


def rollout_batch(bsz=512, L=8192):
    g = torch.Generator(device="cuda").manual_seed(1)
    rlen = torch.randint(1, L + 1, (bsz,), device="cuda", generator=g)
    full = torch.zeros(bsz, 2 * L, dtype=torch.bool, device="cuda")
    full[:, L:] = torch.arange(L, device="cuda")[None] < rlen[:, None]
    return {"advantages": torch.randn(bsz, L, device="cuda", generator=g), "response_mask": full,
            "prompt_lengths": torch.randint(1, 2048, (bsz,), device="cuda", generator=g), "response_lengths": rlen,
            "rewards": torch.randn(bsz, device="cuda", generator=g), "is_end": torch.rand(bsz, device="cuda") < 0.5,
            "values": torch.randn(bsz, L, device="cuda", generator=g)}


def ref_rollout(b, L):
    """compute_rollout_metrics (distributed.py:186-306) restated: collectives counted, .item() reads kept."""
    adv, mask = b["advantages"], b["response_mask"][:, -L:]
    plen, rlen = b["prompt_lengths"], b["response_lengths"]
    plist, dlist = [plen.tolist()], [rlen.tolist()]  # the two all_gather_object calls
    dist.all_gather_into_tensor(torch.empty(2, 1, device="cuda"), torch.zeros(1, device="cuda"))
    dist.all_gather_into_tensor(torch.empty(2, 1, device="cuda"), torch.zeros(1, device="cuda"))
    tdl = torch.tensor(sum(dlist, []))
    sums = [plen.sum().item(), rlen.sum().item(), b["rewards"].sum().item(), b["is_end"].float().sum().item()]
    stats = [tdl.float().mean().item(), tdl.float().var().item(), *(x.item() for x in tdl.float().aminmax())]
    valid = torch.masked_select(adv, mask)
    nv = mask.sum().item()
    sa = valid.double().sum().item()
    red = torch.as_tensor(sums + [sa, plen.numel(), nv], device="cuda", dtype=torch.float32)
    dist.all_reduce(red)
    red = red.tolist()
    mm = torch.as_tensor([-torch.min(valid).item(), torch.max(valid).item()], device="cuda")
    dist.all_reduce(mm)
    v = torch.masked_select(b["values"].float(), mask)
    mv = torch.mean(v)
    dist.all_reduce(mv)
    vm = torch.as_tensor([-torch.min(v).item(), torch.max(v).item()], device="cuda")
    dist.all_reduce(vm)
    return red, mm.tolist(), mv.item(), vm.tolist(), stats, plist


def counted(fake, fn):
    n0 = fake.n
    fn()
    return fake.n - n0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    fake = Counter()
    for name in ("is_available", "is_initialized", "get_world_size", "all_reduce", "all_gather_into_tensor"):
        setattr(dist, name, getattr(fake, name))
    metrics, loss, mask, gvt = epilogue_inputs()
    state = {}

    def ours_mb():
        if state.get("mb", N_MB) == N_MB:
            state["ep"] = MegatronLossEpilogue("actor", num_microbatches=N_MB, early_stop_imp_ratio=10.0,
                                               global_valid_token=gvt)
            state["mb"] = 0
        state["ep"](loss, metrics, mask, state["mb"])
        state["mb"] += 1

    ref_outs = [ref_tail(metrics, loss, mask, gvt)[1] for _ in range(N_MB)]

    def ours_step():
        ep = MegatronLossEpilogue("actor", num_microbatches=N_MB, early_stop_imp_ratio=10.0, global_valid_token=gvt)
        for mb in range(N_MB):
            ep(loss, metrics, mask, mb)
        state["step_ep"] = ep

    ours_step()
    batch = rollout_batch()
    L = batch["advantages"].shape[1]
    cases = {
        "epilogue_per_mb": (ours_mb, lambda: ref_tail(metrics, loss, mask, gvt)),
        "step_finish": (lambda: step_metrics(state["step_ep"]), lambda: ref_step(ref_outs)),
        "rollout_metrics": (lambda: RD.compute_rollout_metrics(batch, 2048, L, return_lengths=False),
                            lambda: ref_rollout(batch, L)),
    }
    res = {}
    for name, (ours, ref) in cases.items():
        for f in (ours, ref):
            f()
        torch.cuda.synchronize()
        t_ours, t_ref = [], []
        for _ in range(args.reps):
            t_ours.append(timed(ours, args.iters))
            t_ref.append(timed(ref, args.iters))
        res[name] = {"ours_ms": statistics.median(t_ours), "ref_ms": statistics.median(t_ref),
                     "ours_syncs": len(host_syncs(ours)), "ref_syncs": len(host_syncs(ref)),
                     "ours_collectives": counted(fake, ours), "ref_collectives": counted(fake, ref)}
    name, plim = card()
    out = {"probe": "reasoning_step", "gpu": name, "power_limit": plim, "rollout_shape": [512, L],
           "epilogue_keys": len(KEYS), "n_mb": N_MB, **res}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
