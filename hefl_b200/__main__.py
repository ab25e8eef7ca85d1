"""Command-line launcher of the product path: multi-round encrypted federated training, one client (or
``--clients-per-rank`` clients) per process (one process per GPU under ``torchrun``; a single process on CPU or one GPU is a 1-client federation).

    # 8 clients on one box, 3 rounds of the reference's medical-CNN recipe (10 local epochs each)
    torchrun --nproc-per-node 8 -m hefl_b200 --rounds 3 --log-jsonl run.jsonl --checkpoint ckpt.pt
    # CPU plumbing config (BASELINE.json configs[0])
    python -m hefl_b200 --device cpu --model cnn2 --image-size 28 --in-channels 1 --num-classes 10 \\
        --he-preset n2048_l1 --nn-backend cudnn --dtype fp32 --rounds 2
    # non-IID hospitals: Dirichlet(0.3) label-skew shards, sample-weighted FedAvg, FedProx mu = 0.01
    torchrun --nproc-per-node 8 -m hefl_b200 --dirichlet-alpha 0.3 --fedavg-weighting samples --fedprox-mu 0.01
    # ... with a server optimizer: FedAdam (eta 0.1, beta1 0.9, beta2 0.99, tau 1e-3) fused into the CKKS decode
    torchrun --nproc-per-node 8 -m hefl_b200 --dirichlet-alpha 0.3 --server-opt fedadam --server-lr 0.1
    # 8 clients on one GPU, half of them sampled per round (DESIGN.md §9)
    python -m hefl_b200 --clients-per-rank 8 --client-fraction 0.5 --dirichlet-alpha 0.3 --fedavg-weighting samples
    # personalised: every client keeps its three Dense layers, 2 head-only epochs before the joint ones (DESIGN.md §10)
    python -m hefl_b200 --clients-per-rank 8 --dirichlet-alpha 0.3 --personal-layers 3 --personal-head-epochs 2
    # after training, class probabilities and a Grad-CAM heatmap of every test scan (DESIGN.md §11)
    python -m hefl_b200 --data-dir image/Train --test-dir image/Test --gradcam-dir cams --gradcam-stage 4
    # after training, pixel-level Integrated Gradients of every test scan, 32 path points (DESIGN.md §12)
    python -m hefl_b200 --data-dir image/Train --test-dir image/Test --ig-dir attributions --ig-steps 32
    # federated evaluation after every round: each client scores its personal model on its shard of image/Test, only
    # the CKKS-summed confusion matrix, ROC histograms and loss sum leave it (DESIGN.md §13)
    python -m hefl_b200 --data-dir image/Train --fed-test-dir image/Test --clients-per-rank 4 --personal-layers 3 \\
        --fed-eval-every 1

Every ``FLConfig`` field is a flag (``--local-epochs 10``) or an environment variable
(``HEFL_LOCAL_EPOCHS=10``); the reference hard-codes all of them (FLPyfhelin.py:31-36, notebook N:24-32).
Extra flags: ``--data-dir DIR`` (the reference's ``image/Train`` layout ``DIR/<label>/<file>``: every rank decodes
its own IID contiguous shard, or with ``--dirichlet-alpha`` its label-skew part of the folder, 10 % of it validates;
without it a synthetic set of the configured shape is used),
``--test-dir DIR`` (same layout; after the last round rank 0 prints the reference's four metrics — weighted
precision / recall / F1 and accuracy, notebook N:267-270 — of the aggregated model; with ``--personal-layers`` of
rank 0's first client's personal model, named by ``"client"``),
``--gradcam-dir DIR`` (needs ``--test-dir``; after the metrics, rank 0 writes ``DIR/predictions.csv`` — file, label,
predicted, p_0 .. p_{C-1} — and one PNG per test scan blended with its Grad-CAM map, then prints
``{"gradcam_dir", "images", "stage"}``), ``--gradcam-stage s`` (the conv stage of the map, default 4),
``--gradcam-class c`` (the explained class; default each scan's predicted class),
``--ig-dir DIR`` (needs ``--test-dir``; after the metrics, rank 0 writes ``DIR/attributions.csv`` — file, label,
target, p_target, score, baseline_score, attribution_sum, gap — and one PNG per test scan blended with its positive
Integrated Gradients attributions, then prints ``{"ig_dir", "images", "steps"}``), ``--ig-steps m`` (path points,
1..1024, default 32), ``--ig-class c`` (the explained class; default each scan's predicted class),
``--fed-test-dir DIR`` (same layout; split among the K clients as ``--data-dir`` is, IID contiguous shards or the
Dirichlet partition under ``--dirichlet-alpha``; each client scores its deployed model on its own shard and only the
CKKS-summed counts leave it; rank 0 prints ``{"round", "fed_eval"}`` after every evaluated round, every
``--fed-eval-every r`` rounds or once after the last round; ``--fed-eval-bins b`` sets the ROC histogram bins),
``--checkpoint PATH`` (written by rank 0 after every round, resumed from if it exists),
``--simulate`` (all ``--clients`` in this one process through the loopback transport: the reference's own
structure, clients as loop iterations, FLPyfhelin.py:184).
"""
from __future__ import annotations

import argparse
import json
import os
import sys


def main(argv=None) -> int:
    import torch
    import torch.distributed as dist

    from .config import FLConfig
    from .fl import FederatedRunner, simulate_clients
    from .utils import StageTimes

    extra = argparse.ArgumentParser(add_help=False)
    extra.add_argument("--checkpoint", default=None)
    extra.add_argument("--data-dir", default=None)
    extra.add_argument("--test-dir", default=None)
    extra.add_argument("--fed-test-dir", default=None)
    extra.add_argument("--stream-decode", action="store_true",
                       help="decode images per batch (flow_from_dataframe semantics) instead of the whole shard up front")
    extra.add_argument("--simulate", action="store_true")
    extra.add_argument("--gradcam-dir", default=None)
    extra.add_argument("--gradcam-stage", type=int, default=4)
    extra.add_argument("--gradcam-class", type=int, default=None)
    extra.add_argument("--ig-dir", default=None)
    extra.add_argument("--ig-steps", type=int, default=32)
    extra.add_argument("--ig-class", type=int, default=None)
    extra.add_argument("-h", "--help", action="store_true")
    ns, rest = extra.parse_known_args(argv)
    if ns.gradcam_dir and not ns.test_dir:
        extra.error("--gradcam-dir explains the scans of --test-dir: give --test-dir DIR as well")
    if ns.ig_dir and not ns.test_dir:
        extra.error("--ig-dir attributes the scans of --test-dir: give --test-dir DIR as well")
    if ns.help:
        print(__doc__)
        print("FLConfig fields:", ", ".join(f.name for f in __import__("dataclasses").fields(FLConfig)))
        return 0
    cfg = FLConfig.from_args(rest)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    use_cuda = cfg.device == "cuda" and torch.cuda.is_available()
    if cfg.device == "cuda" and not use_cuda:
        print("hefl_b200: no CUDA device, falling back to --device cpu --nn-backend cudnn --dtype fp32", file=sys.stderr)
        cfg.device, cfg.nn_backend, cfg.dtype = "cpu", "cudnn", "fp32"
    device = torch.device("cuda", local_rank) if use_cuda else torch.device("cpu")
    if use_cuda:
        torch.cuda.set_device(device)

    if ns.simulate:
        res = simulate_clients(cfg, device=device, rounds=cfg.rounds)
        err = float(res["max_abs_err"]) if "max_abs_err" in res else None
        out = {"mode": "simulate", "clients": cfg.clients, "rounds": cfg.rounds, "max_abs_err_vs_plaintext": err}
        if "global" in res:
            out["server_opt"] = cfg.server_opt
            out["max_abs_err_global_vs_oracle"] = float((res["global"].double() - res["global_oracle"]).abs().max())
        print(json.dumps(out))
        return 0

    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if use_cuda:
            dist.init_process_group("nccl", device_id=device)
        else:
            dist.init_process_group("gloo")
    from .fl.runner import check_client_options, check_personal_options

    check_client_options(cfg)
    check_personal_options(cfg)
    M = cfg.clients_per_rank
    cfg.clients = world * M
    dataset = None
    if ns.data_dir:
        from .fl.data import ImageFolderDataset

        # one shard per client of this rank, in client-id order
        dataset = [ImageFolderDataset(ns.data_dir, cfg.image_size, cfg.in_channels, index=cid, num_clients=cfg.clients,
                                      shuffle_seed=cfg.seed, stream=ns.stream_decode,
                                      dirichlet_alpha=cfg.dirichlet_alpha, min_train=cfg.batch_size)
                   for cid in range(rank * M, rank * M + M)]
        cfg.num_classes = max(cfg.num_classes, dataset[0].classes)
    fed_test = None
    if ns.fed_test_dir:
        from .fl.data import ImageFolderDataset

        # the clients' test shards, split as --data-dir is
        fed_test = [ImageFolderDataset(ns.fed_test_dir, cfg.image_size, cfg.in_channels, index=cid,
                                       num_clients=cfg.clients, shuffle_seed=cfg.seed, stream=ns.stream_decode,
                                       dirichlet_alpha=cfg.dirichlet_alpha)
                    for cid in range(rank * M, rank * M + M)]
    run = FederatedRunner(cfg, rank=rank, world=world, device=device, dataset=dataset, test_dataset=fed_test)
    if ns.gradcam_dir:
        from .fl.explain import check_gradcam

        check_gradcam(run.model, ns.gradcam_stage, ns.gradcam_class, 1)     # before training, not after it
    if ns.ig_dir:
        from .fl.explain import check_ig

        check_ig(run.model, ns.ig_steps, ns.ig_class, 1)
    if ns.checkpoint and os.path.exists(ns.checkpoint):
        run.load_checkpoint(ns.checkpoint)
        if rank == 0:
            print(f"hefl_b200: resumed from {ns.checkpoint} at round {run.round}", file=sys.stderr)
    while run.round < cfg.rounds:
        rec = run.run_round(check=True)
        rec["stage_ms_max"] = StageTimes.max_over_ranks(rec["stage_ms"], device, None)
        run.log.write(rec)
        if rank == 0:
            line = {"round": rec["round"], "loss": rec["loss"], "accuracy": rec["accuracy"],
                    "stage_ms_max": rec["stage_ms_max"], "clients": cfg.clients, "transport": rec["transport"]}
            if "selected" in rec:                    # several clients per rank or client sampling
                line["selected"] = rec["selected"]
                line["rank0_clients"] = rec["clients"]
            print(json.dumps(line))
            if "fed_eval" in rec:
                print(json.dumps({"round": rec["round"], "fed_eval": _fed_line(rec["fed_eval"])}))
        if ns.checkpoint:
            run.save_checkpoint(ns.checkpoint)       # rank 0: global model; every rank: its own optimiser / RNG state
        if world > 1:
            dist.barrier()
    if ns.fed_test_dir and not cfg.fed_eval_every:
        fed = run.evaluate_federated()                  # a collective: every rank
        if rank == 0:
            print(json.dumps({"round": run.round - 1, "fed_eval": _fed_line(fed)}))
    if ns.test_dir and rank == 0:
        from .fl.data import ImageFolderDataset

        test = ImageFolderDataset(ns.test_dir, cfg.image_size, cfg.in_channels, shuffle_seed=None, pin=False)
        if cfg.personal_layers:
            print(json.dumps({"test_images": len(test), "client": run.client_ids[0], **run.evaluate(test, client=0)}))
        else:
            print(json.dumps({"test_images": len(test), **run.evaluate(test)}))
        del test
        if ns.gradcam_dir:
            from .fl.explain import write_explanations

            print(json.dumps(write_explanations(run, ns.test_dir, ns.gradcam_dir, ns.gradcam_stage, ns.gradcam_class,
                                                client=0 if cfg.personal_layers else None)))
        if ns.ig_dir:
            from .fl.explain import write_attributions

            print(json.dumps(write_attributions(run, ns.test_dir, ns.ig_dir, ns.ig_steps, ns.ig_class,
                                                client=0 if cfg.personal_layers else None)))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def _fed_line(fed: dict) -> dict:
    """The federation's evaluation without the rank's own clients' plaintext metrics."""
    return {k: v for k, v in fed.items() if k != "local"}


if __name__ == "__main__":
    sys.exit(main())
