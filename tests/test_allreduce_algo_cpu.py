"""Algorithm choice of the fused all-reduce (``FusedTransport.pick_algo``). The key holder must never take the
one_shot path, where every rank loads every peer's un-aggregated ciphertext, whether one_shot was picked
automatically or forced through ``FLConfig.allreduce_algo`` / ``HEFL_ALLREDUCE_ALGO``. CPU only: the transport
builds on a CPU context at world 1 and its world and key holder are patched in."""
import pytest

from hefl_b200.he.context import CKKSContext
from hefl_b200.parallel import FusedTransport

KB = 1024


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    monkeypatch.delenv("HEFL_ALLREDUCE_ALGO", raising=False)
    monkeypatch.delenv("HEFL_USE_MULTIMEM", raising=False)


def _transport(world, no_owner, algo="auto", mc_ptr=0):
    ctx = CKKSContext(1024, prime_bits=(36,), enforce_security=False)
    t = FusedTransport(ctx, 4096, algo=algo)
    t.world, t.no_owner = world, no_owner
    t.sym.mc_ptr = mc_ptr
    return t


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("nbytes", [4 * KB, 256 * KB, 64 * KB * KB])
def test_forced_algorithm_with_and_without_a_key_holder(world, nbytes):
    for holder in (-1, 0, world // 2, world - 1):
        expect = {"two_shot": "two_shot", "multimem": "multimem",
                  "one_shot": "one_shot" if holder < 0 else "two_shot"}
        for algo, want in expect.items():
            t = _transport(world, holder, algo=algo, mc_ptr=0x1000)
            assert t.pick_algo(nbytes) == want, (world, holder, algo, nbytes)


@pytest.mark.parametrize("algo", ["one_shot", "two_shot", "multimem"])
def test_algorithm_forced_through_the_environment(monkeypatch, algo):
    monkeypatch.setenv("HEFL_ALLREDUCE_ALGO", algo)
    for holder in (-1, 0, 3):
        t = _transport(4, holder, algo="auto", mc_ptr=0x1000)
        assert t.algo == algo
        want = "two_shot" if algo == "one_shot" and holder >= 0 else algo
        assert t.pick_algo(4 * KB) == want, holder


def test_environment_overrides_the_constructor_argument(monkeypatch):
    monkeypatch.setenv("HEFL_ALLREDUCE_ALGO", "one_shot")
    assert _transport(4, 1, algo="two_shot").pick_algo(4 * KB) == "two_shot"
    assert _transport(4, -1, algo="two_shot").pick_algo(4 * KB) == "one_shot"


@pytest.mark.parametrize("world,holder,nbytes,mc,multimem_env,want", [
    (1, -1, 4 * KB, 0, None, "two_shot"),
    (1, -1, 4 * KB, 0x1000, "1", "two_shot"),
    (2, -1, 4 * KB, 0, None, "one_shot"),
    (8, -1, 256 * KB, 0, None, "one_shot"),            # the one_shot threshold is inclusive
    (8, -1, 256 * KB + 32, 0, None, "two_shot"),
    (8, 0, 4 * KB, 0, None, "two_shot"),               # small, but a key holder exists
    (4, 3, 256 * KB, 0, None, "two_shot"),
    (8, -1, 64 * KB * KB, 0x1000, None, "two_shot"),   # multimem only on request
    (8, -1, 64 * KB * KB, 0x1000, "1", "multimem"),
    (8, 0, 4 * KB, 0x1000, "1", "multimem"),           # multimem honours the key holder
    (8, 0, 64 * KB * KB, 0, "1", "two_shot"),          # no multicast object
])
def test_auto_choice(monkeypatch, world, holder, nbytes, mc, multimem_env, want):
    if multimem_env is not None:
        monkeypatch.setenv("HEFL_USE_MULTIMEM", multimem_env)
    assert _transport(world, holder, mc_ptr=mc).pick_algo(nbytes) == want


def test_world_one_has_no_key_holder():
    ctx = CKKSContext(1024, prime_bits=(36,), enforce_security=False)
    t = FusedTransport(ctx, 4096, algo="one_shot", no_owner=0)
    assert t.no_owner == -1 and t.pick_algo(4 * KB) == "one_shot"
