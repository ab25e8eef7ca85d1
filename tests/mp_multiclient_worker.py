"""Multi-process worker: several federated clients per rank. Every rank hosts --clients-per-rank clients, runs
--rounds encrypted FedAvg rounds through FederatedRunner with deterministic crypto and writes the final global model
(rank 0) to --out, so that a test can compare it with the same federation placed differently. gloo (CPU) or nccl
(one GPU per rank, fused transport)."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hefl_b200.config import FLConfig  # noqa: E402
from hefl_b200.fl import FederatedRunner  # noqa: E402


def config(gpu: bool, clients_per_rank: int, client_fraction: float, transport: str) -> FLConfig:
    """The federation both placements run: cnn2 28x28 on CPU, the medical CNN on the tcgen05 engine on GPUs."""
    if gpu:
        return FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=2, val_steps=1, nn_backend="tcgen05",
                        transport=transport, device="cuda", deterministic_crypto=True, key_holder=-1,
                        clients_per_rank=clients_per_rank, client_fraction=client_fraction)
    return FLConfig(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                    steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32",
                    transport=transport, device="cpu", deterministic_crypto=True, key_holder=-1,
                    clients_per_rank=clients_per_rank, client_fraction=client_fraction)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--clients-per-rank", type=int, default=2)
    ap.add_argument("--client-fraction", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", required=True)
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
    cfg = config(gpu, args.clients_per_rank, args.client_fraction, "fused" if gpu else "gloo")
    run = FederatedRunner(cfg, rank=rank, world=world, device=device)
    selected = []
    for _ in range(args.rounds):
        rec = run.run_round(check=True)
        selected.append(rec["selected"])
    ref = run.pack.flat.clone()
    dist.broadcast(ref, src=0)
    assert torch.equal(ref, run.pack.flat), "ranks diverged"
    if rank == 0:
        torch.save(run.pack.flat.cpu(), args.out)
        print("MP_REPORT " + json.dumps({"world": world, "transport": run.transport.name, "selected": selected}))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
