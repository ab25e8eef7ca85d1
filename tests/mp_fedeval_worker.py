"""Multi-process worker: federated evaluation over gloo with a key holder and pairwise masks. Every rank hosts
--clients-per-rank clients, each with its own test set (``test_sets``), runs one round with fed_eval_every = 1 and
deterministic crypto, and writes the round's ``fed_eval`` to ``--out.rank{r}``, so that a test can compare it with the
same federation placed in one process."""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hefl_b200.config import FLConfig  # noqa: E402
from hefl_b200.fl import FederatedRunner  # noqa: E402
from hefl_b200.fl.data import SyntheticImageDataset  # noqa: E402

SIZES = (11, 0, 17, 6)        # test scans of clients 0..3


def config(clients_per_rank: int, transport: str, key_holder: int) -> FLConfig:
    return FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                    steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32",
                    transport=transport, device="cpu", deterministic_crypto=True, key_holder=key_holder,
                    pairwise_masks=key_holder >= 0, clients_per_rank=clients_per_rank, fed_eval_every=1,
                    fed_eval_bins=20)


def test_sets(ids):
    return [SyntheticImageDataset(SIZES[c], 28, 1, 10, seed=300 + c, pin=False) for c in ids]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients-per-rank", type=int, default=2)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    M = args.clients_per_rank
    run = FederatedRunner(config(M, "gloo", 0), rank=rank, world=world, device=torch.device("cpu"),
                          test_dataset=test_sets(range(rank * M, rank * M + M)))
    rec = run.run_round(check=True)
    torch.save({k: v for k, v in rec["fed_eval"].items() if k != "local"}, f"{args.out}.rank{rank}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
