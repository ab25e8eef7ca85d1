"""Multi-process tests. CPU (gloo, world 2) checks the host-side transport logic here;
the GPU variants run the fused NVLink kernel across real devices on an H100 and skip on a one-GPU machine.
test_gpu_allreduce_ranks.py runs the same kernel with 1-8 logical ranks in one process on one GPU."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "mp_allreduce_worker.py")


FED_WORKER = os.path.join(ROOT, "tests", "mp_fedavg_worker.py")


def _run(nproc, backend, port, extra=(), worker=None):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), worker or WORKER, "--backend", backend, *extra]
    env = dict(os.environ, OMP_NUM_THREADS="2")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("MP_REPORT ")][-1]
    return json.loads(line[len("MP_REPORT "):])


def test_collective_transport_gloo_world2():
    rep = _run(2, "gloo", 29611, ["--rounds", "2", "--cts", "3"])
    assert rep["world"] == 2 and rep["checks"] == 2


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_fused_allreduce_across_gpus(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    rep = _run(nproc, "nccl", 29620 + nproc)
    assert rep["world"] == nproc and rep["checks"] >= 5 + 2 * 6


def test_federated_round_gloo_world2():
    """Whole product path on two CPU ranks: local training, CKKS encrypt, all-reduce, decrypt."""
    rep = _run(2, "gloo", 29641, ["--rounds", "2"], worker=FED_WORKER)
    assert rep["world"] == 2 and rep["max_abs_err"] < 1e-5


def test_federated_round_with_a_dropped_client_gloo():
    """allow_dropouts: rank 1 sits the rounds out (encrypts zeros); K = 1 is agreed at run time and the
    aggregate equals the mean over the participating clients on every rank."""
    rep = _run(2, "gloo", 29645, ["--rounds", "2", "--drop-rank", "1"], worker=FED_WORKER)
    assert rep["world"] == 2 and rep["max_abs_err"] < 1e-5


def test_federated_round_with_pairwise_masks_gloo():
    """pairwise_masks: X25519-agreed PRG masks on every client's ciphertext cancel in the all-reduce."""
    rep = _run(2, "gloo", 29647, ["--rounds", "2", "--masks", "--key-holder", "0"], worker=FED_WORKER)
    assert rep["world"] == 2 and rep["max_abs_err"] < 1e-5


def test_federated_round_with_a_single_key_holder_gloo():
    """key_holder=1: only rank 1 keeps the secret key, decrypts and broadcasts; same result on every rank."""
    rep = _run(2, "gloo", 29643, ["--rounds", "2", "--key-holder", "1"], worker=FED_WORKER)
    assert rep["world"] == 2 and rep["max_abs_err"] < 1e-5


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("nproc,model", [(2, "cnn2"), (2, "medcnn"), (8, "medcnn")])
def test_federated_round_across_gpus(nproc, model):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    rep = _run(nproc, "nccl", 29650 + nproc, ["--rounds", "2", "--model", model], worker=FED_WORKER)
    assert rep["transport"] == "fused" and rep["max_abs_err"] < 1e-5


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("nproc", [2, 8])
def test_key_holder_never_loads_peer_ciphertext_across_gpus(nproc):
    """Default trust model on the fused transport: rank 0 generates the keys, owns no chunk of the all-reduce
    (its peer-load counter stays 0 while every other rank's is positive), decrypts and broadcasts; with masks."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    rep = _run(nproc, "nccl", 29670 + nproc, ["--rounds", "2", "--model", "medcnn", "--key-holder", "0", "--masks"],
               worker=FED_WORKER)
    assert rep["transport"] == "fused" and rep["max_abs_err"] < 1e-5
