"""The chunked FedAvg round on CPU tensors (cnn2 28x28, n = 2048 / one prime: six ciphertexts, two of the shared base
with a personal layer, three at n = 4096 for the server step; loopback transport):
``fedavg_pipelined`` at every chunk size installs, bit for bit, what ``encrypt_update -> aggregate ->
decrypt_apply`` installs, and leaves the same server-optimizer state."""
import pytest
import torch

from hefl_b200.config import FLConfig
from hefl_b200.fl import FederatedRunner

CPU = torch.device("cpu")


def _cfg(**kw):
    base = dict(model="cnn2", image_size=28, in_channels=1, num_classes=10, batch_size=8, local_epochs=1,
                steps_per_epoch=2, val_steps=1, he_preset="n2048_l1", nn_backend="cudnn", dtype="fp32", device="cpu",
                transport="loopback", deterministic_crypto=True, key_holder=-1)
    base.update(kw)
    return FLConfig(**base)


CASES = {
    "fedavg": {},
    "fedadam": dict(server_opt="fedadam", server_lr=0.1, he_preset="n4096_l3"),
    "personal": dict(personal_layers=1),
    "two_clients": dict(clients_per_rank=2),
    "nobody": dict(allow_dropouts=True),
}


def _two_rounds(cfg, chunk_cts=None):
    """A fresh runner through two rounds; ``chunk_cts`` None takes the unchunked stages. Returns the runner and
    the model its last round trained, before that round's FedAvg."""
    run = FederatedRunner(cfg, device=CPU)
    run.participating = not cfg.allow_dropouts           # "nobody": every client sits both rounds out
    for _ in range(2):
        run.global_flat.copy_(run.pack.flat)
        run.local_train()
        trained = run.pack.flat.clone()
        if chunk_cts is None:
            run.decrypt_apply(run.aggregate(run.encrypt_update()))
        else:
            run.fedavg_pipelined(chunk_cts=chunk_cts)
        run.round += 1
    return run, trained


@pytest.mark.parametrize("case", list(CASES))
def test_every_chunk_size_installs_the_unchunked_model(case):
    cfg = _cfg(**CASES[case])
    ref, trained = _two_rounds(cfg)
    if case == "nobody":
        assert torch.equal(ref.pack.flat, trained), "a round nobody took part in changed the model"
    else:
        assert not torch.equal(ref.shared(), trained[: ref.n_shared])
    assert ref.n_ct >= 2                                  # chunk_cts=1 splits the round
    for c in range(1, ref.n_ct + 1):
        run, trained = _two_rounds(cfg, chunk_cts=c)
        if case == "nobody":
            assert torch.equal(run.pack.flat, trained), f"chunk_cts={c}: a round nobody took part in changed the model"
        assert torch.equal(run.pack.flat, ref.pack.flat), f"chunk_cts={c}: the model differs"
        if ref.server_opt is not None:
            assert torch.equal(run.server_opt.m, ref.server_opt.m), f"chunk_cts={c}: server m differs"
            assert torch.equal(run.server_opt.v, ref.server_opt.v), f"chunk_cts={c}: server v differs"
