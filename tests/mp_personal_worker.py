"""Multi-process worker: personalised federated learning over gloo. Every rank hosts --clients-per-rank clients that
keep their last --personal-layers Dense layers, runs --rounds rounds with deterministic crypto and writes its shared
base and its clients' personal layers to ``--out.rank{r}``, so that a test can compare them with the same federation
placed in one process."""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hefl_b200.config import FLConfig  # noqa: E402
from hefl_b200.fl import FederatedRunner  # noqa: E402


def config(clients_per_rank: int, transport: str) -> FLConfig:
    """cnn2 28x28 on CPU; its one Dense layer is personal and trains one head-only epoch before the joint one."""
    return FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                    steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32",
                    transport=transport, device="cpu", deterministic_crypto=True, key_holder=-1,
                    clients_per_rank=clients_per_rank, personal_layers=1, personal_head_epochs=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients-per-rank", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    run = FederatedRunner(config(args.clients_per_rank, "gloo"), rank=rank, world=world, device=torch.device("cpu"))
    for _ in range(args.rounds):
        run.run_round(check=True)
    base = run.shared().clone()
    ref = base.clone()
    dist.broadcast(ref, src=0)
    assert torch.equal(ref, base), "ranks diverged"
    torch.save({"ids": run.client_ids, "base": base, "heads": run._heads().clone()}, f"{args.out}.rank{rank}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
