"""Multi-process worker for non-IID encrypted FedAvg: Dirichlet label-skew shards, sample-weighted aggregation and
the FedProx term on every rank. Checks that the decrypted aggregate equals sum(n_k x_k) / N of the ranks' locally
trained weights (the participants' only, with a rank sitting out), that every rank ends with the same model, and
that the runner's own debug_precision oracle agrees. gloo (CPU) or nccl (one GPU per rank)."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hefl_b200.config import FLConfig  # noqa: E402
from hefl_b200.fl import FederatedRunner  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--model", default="cnn2")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--drop-rank", type=int, default=-1)
    ap.add_argument("--alpha", type=float, default=0.3)
    ap.add_argument("--mu", type=float, default=0.01)
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
    common = dict(clients=world, dirichlet_alpha=args.alpha, fedavg_weighting="samples", fedprox_mu=args.mu,
                  allow_dropouts=args.drop_rank >= 0, key_holder=0, local_epochs=1)
    if args.model == "medcnn":
        cfg = FLConfig(model="medcnn", steps_per_epoch=3, val_steps=1, nn_backend="tcgen05" if gpu else "cudnn",
                       transport="fused" if gpu else "gloo", device="cuda" if gpu else "cpu", **common)
    else:
        cfg = FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, steps_per_epoch=4,
                       val_steps=1, he_preset="n4096_l3", nn_backend="cudnn", dtype="bf16" if gpu else "fp32",
                       transport="fused" if gpu else "gloo", device="cuda" if gpu else "cpu", **common)
    run = FederatedRunner(cfg, rank=rank, world=world, device=device)
    run.participating = rank != args.drop_rank
    sizes = [torch.zeros(1, dtype=torch.float64, device=device) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([float(run.n_train)], dtype=torch.float64, device=device))
    sizes = [int(s.item()) for s in sizes]
    worst = 0.0
    weights = []
    for rnd in range(args.rounds):
        run.local_train()
        mine = run.pack.flat.clone()
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        keep = [r for r in range(world) if r != args.drop_rank]
        n_tot = sum(sizes[r] for r in keep)
        oracle = sum(sizes[r] * gathered[r].double() for r in keep) / n_tot
        ct = run.encrypt_update()
        weights.append(run.fedavg_weight())
        run.decrypt_apply(run.aggregate(ct))
        run.guard_finite()
        err = float((run.pack.flat.double() - oracle).abs().max())
        worst = max(worst, err)
        ref = run.pack.flat.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(ref, run.pack.flat), "ranks diverged"
        if args.drop_rank >= 0:
            # K = 1: the survivor's weight is exactly 1 and the aggregate is its model
            assert weights[-1] == 1.0 or rank == args.drop_rank
        run.round += 1
    # the runner's own plaintext oracle (debug_precision) over one more full round
    run.cfg.debug_precision = True
    rec = run.run_round(check=True)
    t = torch.tensor([worst, rec["ckks_max_abs_err"]], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print("MP_REPORT " + json.dumps({"world": world, "transport": run.transport.name, "n_train": sizes,
                                         "weights_rank0": weights, "max_abs_err": float(t[0]),
                                         "debug_precision_err": float(t[1]), "fedavg_weight": rec["fedavg_weight"],
                                         "label_counts": rec["label_counts"]}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
