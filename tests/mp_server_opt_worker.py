"""Multi-process worker for the server optimizer of encrypted FedAvg (DESIGN.md §8). With a key holder, only that
rank holds server state, steps the model in the fused decode and broadcasts it: every rank must end every round
with the key holder's model bit for bit. With key_holder = -1 every rank decrypts and applies the same
deterministic step: the models and the states must agree bit for bit after every round. The last round runs with
debug_precision, whose error must describe the decoded average. gloo (CPU) or nccl (one GPU per rank)."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hefl_b200.config import FLConfig  # noqa: E402
from hefl_b200.fl import FederatedRunner  # noqa: E402


def same_on_all_ranks(t: torch.Tensor) -> bool:
    ref = t.clone()
    dist.broadcast(ref, src=0)
    ok = torch.tensor([1 if torch.equal(ref, t) else 0], device=t.device)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    return bool(int(ok))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--model", default="cnn2")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--key-holder", type=int, default=0)
    ap.add_argument("--opt", default="fedadam")
    args = ap.parse_args()
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
    gpu = args.backend == "nccl"
    if gpu:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        device = torch.device("cuda", torch.cuda.current_device())
        dist.init_process_group("nccl", device_id=device)
    else:
        device = torch.device("cpu")
        dist.init_process_group("gloo")
    common = dict(clients=world, key_holder=args.key_holder, local_epochs=1, server_opt=args.opt, server_lr=0.1,
                  dirichlet_alpha=0.5, fedavg_weighting="samples")
    if args.model == "medcnn":
        cfg = FLConfig(model="medcnn", steps_per_epoch=3, val_steps=1, nn_backend="tcgen05" if gpu else "cudnn",
                       transport="fused" if gpu else "gloo", device="cuda" if gpu else "cpu", **common)
    else:
        cfg = FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, steps_per_epoch=4,
                       val_steps=1, he_preset="n4096_l3", nn_backend="cudnn", dtype="bf16" if gpu else "fp32",
                       transport="fused" if gpu else "gloo", device="cuda" if gpu else "cpu", **common)
    run = FederatedRunner(cfg, rank=rank, world=world, device=device)
    rounds_equal = state_equal = 0
    err = float("nan")
    for rnd in range(args.rounds):
        run.cfg.debug_precision = rnd == args.rounds - 1
        x0 = run.pack.flat.clone()
        rec = run.run_round(check=True)
        assert rec["server_opt"] == args.opt
        assert not torch.equal(run.pack.flat, x0)
        rounds_equal += same_on_all_ranks(run.pack.flat)
        if run.server_opt is not None and args.key_holder < 0:
            state_equal += same_on_all_ranks(run.server_opt.m) and same_on_all_ranks(run.server_opt.v)
        if "ckks_max_abs_err" in rec:
            err = rec["ckks_max_abs_err"]
    on = torch.tensor([1.0 if run.server_opt is not None else 0.0], device=device)
    ons = [torch.zeros_like(on) for _ in range(world)]
    dist.all_gather(ons, on)
    t = torch.tensor([err], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print("MP_REPORT " + json.dumps({"world": world, "transport": run.transport.name, "rounds": args.rounds,
                                         "rounds_equal": rounds_equal, "state_equal": state_equal,
                                         "state_on": [bool(float(o)) for o in ons],
                                         "debug_precision_err": float(t[0])}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
