"""The fused ciphertext all-reduce (csrc/comm/allreduce_modq.cu) at every world size, on one GPU.

W logical ranks live in this process. Each has its own buffer (and one_shot output), signal pad, status word,
stats word and stream, and the W launches run concurrently and meet at the kernel's cross-rank block barriers
as W GPUs would. That reaches every instantiation of the kernel (U = 4, 2, 1 for worlds 1-2, 3-4, 5-8), the
key holder, 61-bit primes, views at an offset into the buffer, and the pairwise-mask and local-sum kernels.

References: every limb is summed as ``acc = (acc + x_r) % q`` in int64, one rank at a time (no value exceeds
2^62), and the chunk partition is written out from its documented rule. Neither uses the Barrett constants the
kernel reduces with.

Co-residency: the block barriers only meet if every CTA of every rank is resident at once. The kernel takes
at most one CTA per SM at 512 threads, so ``W x blocks`` is kept at or below half the SMs at any thread count
(even grids are launched as clusters of two and must find whole free TPCs). All spins are bounded, so a
violation shows up as a nonzero status word after TIMEOUT_MS, not as a hang.

Launch order: every rank's launch i is enqueued before any rank's launch i + 1. Streams share a limited number
of hardware queues, and a rank's later work queued ahead of a peer's launch that its own earlier launch waits
for would stall both until the timeout.
"""
import functools
import hashlib
import os
import types

import pytest
import torch

from hefl_b200 import _ext
from hefl_b200.he.context import CKKSContext
from hefl_b200.parallel import FusedTransport

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(os.environ.get("CUDA_LAUNCH_BLOCKING") == "1",
                       reason="serialised launches: the logical ranks' kernels could never meet at their barriers"),
]
ops = _ext.ops()

ALGO = {"two_shot": 0, "one_shot": 1}
TIMEOUT_MS = 5000
SENTINEL = 0x5A5A5A5A5A5A5A5A          # not a residue of any prime used here: a stray write changes it


# ---------------------------------------------------------------------------------------------- references
@functools.lru_cache(maxsize=None)
def _ctx(logn, bits, L):
    return CKKSContext(1 << logn, prime_bits=(bits,) * L, scale_bits=30, enforce_security=False)


def q_of_word(primes, numel, logn):
    """The prime of every word of a flat [C][2][L][N] buffer: word e lies in limb (e >> logn) % L."""
    return torch.tensor(primes, dtype=torch.int64)[(torch.arange(numel) >> logn) % len(primes)]


def residues(qw, gen):
    """Uniform residues with q - 1 and 0 sprinkled in."""
    x = torch.randint(0, 2 ** 62, qw.shape, generator=gen, dtype=torch.int64) % qw
    x[::5] = qw[::5] - 1
    x[1::11] = 0
    return x


def land_sums_near_multiples_of_q(inputs, qw, sel):
    """Pick the last rank's words at ``sel`` so that the plain sum over ranks is a multiple of q plus 0..3. Barrett's
    quotient falls one short exactly there, so these words need the reduction's correction step."""
    others = ref_sum(inputs[:-1], qw)[sel]
    t = torch.arange(qw.numel())[sel] % 4
    inputs[-1][sel] = (t - others) % qw[sel]


def ref_sum(inputs, qw):
    acc = torch.zeros_like(qw)
    for x in inputs:
        acc = (acc + x) % qw
    return acc


def owner_ranges(quads, world, holder=-1):
    """[lo, hi) quads of every rank: owners are all ranks but the key holder, renumbered in rank order;
    per = ceil(quads / owners); owner m gets [min(m per, quads), min(m per + per, quads)); the holder gets none."""
    owners = [r for r in range(world) if r != holder]
    per = -(-quads // len(owners))
    rng = {holder: (0, 0)}
    for m, r in enumerate(owners):
        rng[r] = (min(m * per, quads), min(m * per + per, quads))
    return [rng[r] for r in range(world)]


def unroll(world):
    """Quads per thread per step of the P2P instantiation a world size launches."""
    return 4 if world <= 2 else 2 if world <= 4 else 1


def awkward_numel(full, owners, step):
    """The largest word count <= full whose quads split unevenly among the owners (if more than one) and give
    no owner a range that is a whole number of kernel steps (blocks x threads x unroll quads)."""
    for numel in range(full, full - 4 * 512, -4):
        quads = numel // 4
        if owners > 1 and quads % owners == 0:
            continue
        if any(hi > lo and (hi - lo) % step == 0 for lo, hi in owner_ranges(quads, owners)):
            continue
        return numel
    raise AssertionError("no awkward size found")


def pair_seed(i, j, seed=1234):
    """A 63-bit pair seed, derived as the runner's deterministic path derives it."""
    h = hashlib.sha256(f"hefl-pair-{seed}-{min(i, j)}-{max(i, j)}".encode()).digest()
    return int.from_bytes(h[:8], "little") >> 1


def assert_words(got, exp, what):
    got, exp = got.cpu(), exp.cpu()
    if not torch.equal(got, exp):
        bad = (got != exp).nonzero().flatten()
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.numel()} of {exp.numel()} words differ, the first at word {i}: "
                             f"got {int(got[i]) & (2**64 - 1):#x}, expected {int(exp[i]) & (2**64 - 1):#x}")


# ---------------------------------------------------------------------------------------------- harness
def cta_budget():
    """CTAs all ranks together may launch (see the module docstring)."""
    return torch.cuda.get_device_properties(0).multi_processor_count // 2


def grid(world, parity, cap=16):
    b = min(cap, cta_budget() // world)
    if b % 2 != parity:
        b -= 1
    assert b >= 1 and world * b <= cta_budget()
    return b


class Ranks:
    """W logical ranks on this GPU. Buffers and outputs start filled with SENTINEL."""

    def __init__(self, world, words, max_blocks):
        dev = "cuda"
        self.world = world
        self.bufs = [torch.full((words,), SENTINEL, dtype=torch.int64, device=dev) for _ in range(world)]
        self.outs = [torch.full((words,), SENTINEL, dtype=torch.int64, device=dev) for _ in range(world)]
        self.sigs = [torch.zeros(2 * max_blocks * world + 64, dtype=torch.int32, device=dev) for _ in range(world)]
        self.status = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(world)]
        self.stats = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(world)]
        self.streams = [torch.cuda.Stream() for _ in range(world)]

    def load(self, inputs, off=0):
        for b, x in zip(self.bufs, inputs):
            b[off:off + x.numel()].copy_(x)
        torch.cuda.synchronize()

    def launch(self, r, algo, ctx, logn, numel, blocks, threads, off=0, holder=-1):
        with torch.cuda.stream(self.streams[r]):
            ops.allreduce_modq([b.data_ptr() + 8 * off for b in self.bufs], [s.data_ptr() for s in self.sigs], 0,
                               self.outs[r][off:off + numel] if algo == "one_shot" else None, self.status[r],
                               ctx.consts_cpu, numel, ctx.L, logn, r, self.world, ALGO[algo], blocks, threads,
                               TIMEOUT_MS, holder, self.stats[r])

    def run(self, algo, ctx, logn, numel, blocks, threads, off=0, holder=-1):
        for r in range(self.world):
            self.launch(r, algo, ctx, logn, numel, blocks, threads, off, holder)
        self.finish()

    def finish(self):
        torch.cuda.synchronize()
        for r in range(self.world):
            code = int(self.status[r].item())
            assert code == 0, (f"rank {r} timed out at a block barrier (status {code:#x}): were all CTAs of all "
                               f"{self.world} ranks co-resident?")
        for r in range(self.world):
            assert int(self.sigs[r].abs().sum().item()) == 0, f"rank {r}: signal pad did not return to rest"

    def result(self, r, algo, off, numel):
        return (self.outs[r] if algo == "one_shot" else self.bufs[r])[off:off + numel]

    def take_stats(self):
        s = [int(t.item()) for t in self.stats]
        for t in self.stats:
            t.zero_()
        return s


def check_stats(steps, quads, world, holder, algo):
    """Peer-load steps are counted per 32-byte quad: a two_shot owner's range length, a one_shot rank's all quads,
    the key holder's none."""
    if algo == "one_shot":
        assert steps == [quads] * world, steps
        return
    want = [hi - lo for lo, hi in owner_ranges(quads, world, holder)]
    assert steps == want, (steps, want)
    assert sum(steps) == quads


# ---------------------------------------------------------------------------------------------- (a)
CASES_A = [(bits, L, logn) for bits in (36, 61) for L in (1, 3, 5) for logn in (10, 12)]


@pytest.mark.parametrize("algo", ["two_shot", "one_shot"])
@pytest.mark.parametrize("world", range(1, 9))
def test_every_world_size_and_instantiation(world, algo):
    """Worlds 1-8 reach all three unroll instantiations. Sizes are chosen so that the quads split unevenly and no
    rank's range is a whole number of kernel steps; grids are odd (no clusters) and even (clusters of two)."""
    gen = torch.Generator().manual_seed(100 * world + ALGO[algo])
    for i, (bits, L, logn) in enumerate(CASES_A):
        parity, threads = i % 2, (32, 128, 512)[i % 3]
        blocks = grid(world, parity)
        ctx = _ctx(logn, bits, L)
        owners = world if algo == "two_shot" else 1
        step = blocks * threads * unroll(world)
        quads_per_ct = L << (logn - 1)
        C = max(1, -(-(step * owners * 5 // 2) // quads_per_ct))      # about 2.5 steps per owner
        numel = awkward_numel(C * 2 * L << logn, owners, step)
        what = f"world {world} {algo} {bits}-bit L={L} logn={logn} numel={numel} grid {blocks}x{threads}"
        qw = q_of_word(ctx.primes, numel, logn)
        inputs = [residues(qw, gen) for _ in range(world)]
        land_sums_near_multiples_of_q(inputs, qw, slice(2, None, 3))
        exp = ref_sum(inputs, qw)
        ranks = Ranks(world, numel, blocks)
        ranks.load(inputs)
        ranks.run(algo, ctx, logn, numel, blocks, threads)
        for r in range(world):
            assert_words(ranks.result(r, algo, 0, numel), exp, f"{what}: rank {r}")
            if algo == "one_shot":
                assert_words(ranks.bufs[r], inputs[r], f"{what}: rank {r} input")
        check_stats(ranks.take_stats(), numel // 4, world, -1, algo)


# ---------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("world", range(2, 9))
def test_key_holder_owns_no_chunk_and_receives_the_sum(world):
    gen = torch.Generator().manual_seed(world)
    for holder in sorted({0, world // 2, world - 1}):
        for bits, L, logn, C, threads, parity in ((61, 3, 12, 3, 512, 0), (36, 5, 10, 4, 128, 1)):
            ctx = _ctx(logn, bits, L)
            blocks = grid(world, parity)
            numel = C * 2 * L << logn
            qw = q_of_word(ctx.primes, numel, logn)
            inputs = [residues(qw, gen) for _ in range(world)]
            exp = ref_sum(inputs, qw)
            ranks = Ranks(world, numel, blocks)
            ranks.load(inputs)
            ranks.run("two_shot", ctx, logn, numel, blocks, threads, holder=holder)
            for r in range(world):
                assert_words(ranks.bufs[r], exp, f"world {world} holder {holder} {bits}-bit: rank {r}")
            steps = ranks.take_stats()
            assert steps[holder] == 0, f"the key holder issued {steps[holder]} peer-load steps"
            check_stats(steps, numel // 4, world, holder, "two_shot")


def test_tiny_buffer_leaves_some_owners_without_a_range():
    world, holder, numel, logn = 8, 0, 36, 12
    ranges = owner_ranges(numel // 4, world, holder)
    assert [hi - lo for lo, hi in ranges].count(0) == 3                  # the holder and two empty owners
    ctx = _ctx(logn, 61, 3)
    gen = torch.Generator().manual_seed(8)
    qw = q_of_word(ctx.primes, numel, logn)
    inputs = [residues(qw, gen) for _ in range(world)]
    ranks = Ranks(world, numel, 1)
    ranks.load(inputs)
    ranks.run("two_shot", ctx, logn, numel, 1, 32, holder=holder)
    for r in range(world):
        assert_words(ranks.bufs[r], ref_sum(inputs, qw), f"rank {r}")
    check_stats(ranks.take_stats(), numel // 4, world, holder, "two_shot")


def make_transports(ctx, world, max_numel, holder, algo="auto", blocks=None):
    """W world-1 FusedTransports rewired into one W-rank group on this GPU."""
    ts = [FusedTransport(ctx, max_numel, algo=algo, timeout_s=TIMEOUT_MS / 1000) for _ in range(world)]
    # signal pads need 2 * max_blocks * W + 64 flags; the world-1 ones only have room for one rank
    sigs = [torch.zeros(2 * ts[0].max_blocks * world + 64, dtype=torch.int32, device="cuda") for _ in range(world)]
    ptrs = [t.sym.tensor.data_ptr() for t in ts]
    for r, t in enumerate(ts):
        t.world, t.rank, t.no_owner = world, r, holder
        t.sym.ptrs, t.sym.mc_ptr = list(ptrs), 0
        t.sig = types.SimpleNamespace(tensor=sigs[r], ptrs=[s.data_ptr() for s in sigs])
        t.blocks = blocks or cta_budget() // world
    return ts


def transport_round(ts, streams, chunks, per_ct, shape_tail):
    """Every rank all-reduces the views buf[c0 per_ct : c1 per_ct] of its symmetric buffer, chunk after chunk."""
    for c0, c1 in chunks:
        for t, st in zip(ts, streams):
            with torch.cuda.stream(st):
                t.allreduce(t.sym.tensor[c0 * per_ct: c1 * per_ct].view(c1 - c0, *shape_tail))
    torch.cuda.synchronize()
    for t in ts:
        t.check_status()


@pytest.mark.parametrize("world,holder", [(2, 0), (3, 2), (8, 0), (8, 5)])
def test_forced_one_shot_keeps_the_key_holder_off_peer_ciphertext(monkeypatch, world, holder):
    """FLConfig.allreduce_algo / HEFL_ALLREDUCE_ALGO = one_shot with a key holder: the transport runs two_shot and
    the holder loads nothing."""
    monkeypatch.delenv("HEFL_ALLREDUCE_ALGO", raising=False)
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, enforce_security=False, device="cuda")
    C, L, n = 3, ctx.L, ctx.n
    per_ct = 2 * L * n
    ts = make_transports(ctx, world, C * per_ct, holder, algo="one_shot")
    gen = torch.Generator().manual_seed(world)
    qw = q_of_word(ctx.primes, C * per_ct, ctx.logn)
    inputs = [residues(qw, gen) for _ in range(world)]
    for t, x in zip(ts, inputs):
        t.sym.tensor.copy_(x)
    torch.cuda.synchronize()
    transport_round(ts, [torch.cuda.Stream() for _ in ts], [(0, C)], per_ct, (2, L, n))
    exp = ref_sum(inputs, qw)
    for r, t in enumerate(ts):
        assert t.last_algo == "two_shot"
        assert_words(t.sym.tensor, exp, f"rank {r}")
    steps = [t.peer_load_steps() for t in ts]
    assert steps[holder] == 0, f"the key holder loaded {steps[holder]} quads of its peers' ciphertext"
    check_stats(steps, C * per_ct // 4, world, holder, "two_shot")


# ---------------------------------------------------------------------------------------------- (c)
@pytest.mark.parametrize("algo,holder", [("two_shot", -1), ("one_shot", -1), ("two_shot", 0)])
def test_largest_sums_just_below_2_64(algo, holder):
    """Eight residues of q - 1 under a 61-bit prime sum to just below 2^64: the kernel's u64 sum must not wrap,
    and its reduction must be exact right up to there."""
    world, logn, L = 8, 12, 3
    ctx = _ctx(logn, 61, L)
    assert all(2 ** 63 < world * (q - 1) < 2 ** 64 for q in ctx.primes)
    numel = 4 * 2 * L << logn
    qw = q_of_word(ctx.primes, numel, logn)
    gen = torch.Generator().manual_seed(61)
    inputs = []
    half = numel // 2
    for _ in range(world):
        x = qw - 1                                                           # first half: q - 1 on every rank
        pick = torch.randint(0, 3, (numel - half,), generator=gen)
        near = qw[half:] - 1 - torch.randint(0, 2 ** 40, (numel - half,), generator=gen, dtype=torch.int64)
        x[half:] = torch.where(pick == 0, qw[half:] - 1, torch.where(pick == 1, torch.zeros_like(near), near))
        inputs.append(x)
    land_sums_near_multiples_of_q(inputs, qw, slice(half + 1, None, 3))
    exp = ref_sum(inputs, qw)
    assert torch.equal(exp[:half], qw[:half] - world)
    blocks = grid(world, 1)
    ranks = Ranks(world, numel, blocks)
    ranks.load(inputs)
    ranks.run(algo, ctx, logn, numel, blocks, 256, holder=holder)
    for r in range(world):
        assert_words(ranks.result(r, algo, 0, numel), exp, f"{algo} holder {holder}: rank {r}")


# ---------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("world,algo,holder,bits", [(3, "two_shot", -1, 36), (8, "two_shot", 0, 61),
                                                    (5, "one_shot", -1, 61), (8, "one_shot", -1, 36)])
def test_offset_views_and_back_to_back_launches(world, algo, holder, bits):
    """The pipeline's layout: chunk views buf[c0 per_ct : c1 per_ct] reduced one after another on each rank's
    stream; the words outside the views stay untouched on every rank. Then 20 launches per rank with no host
    synchronisation, each rank re-copying its input on its own stream before each launch."""
    logn, L, n_ct = 12, 3, 7
    ctx = _ctx(logn, bits, L)
    per_ct = 2 * L << logn
    words = n_ct * per_ct
    chunks = [(1, 3), (3, 4), (4, 6)]                 # ciphertexts 0 and 6 are never part of a view
    lo, hi = chunks[0][0] * per_ct, chunks[-1][1] * per_ct
    qw = q_of_word(ctx.primes, words, logn)[lo:hi]
    gen = torch.Generator().manual_seed(world)
    sets = [[residues(qw, gen) for _ in range(world)] for _ in range(2)]
    exps = [ref_sum(s, qw) for s in sets]
    blocks, threads = grid(world, 0), 128
    ranks = Ranks(world, words, blocks)
    ranks.load(sets[0], off=lo)
    sentinel = torch.full((words,), SENTINEL, dtype=torch.int64)

    def check(exp, inputs, what):
        for r in range(world):
            res = ranks.result(r, algo, 0, words).cpu()
            assert_words(res[lo:hi], exp, f"{what}: rank {r}")
            assert_words(torch.cat([res[:lo], res[hi:]]), torch.cat([sentinel[:lo], sentinel[hi:]]),
                         f"{what}: rank {r} outside the views")
            if algo == "one_shot":
                buf = ranks.bufs[r].cpu()
                assert_words(buf[lo:hi], inputs[r], f"{what}: rank {r} input")
                assert_words(torch.cat([buf[:lo], buf[hi:]]), torch.cat([sentinel[:lo], sentinel[hi:]]),
                             f"{what}: rank {r} buffer outside the views")

    for c0, c1 in chunks:
        for r in range(world):
            ranks.launch(r, algo, ctx, logn, (c1 - c0) * per_ct, blocks, threads, off=c0 * per_ct, holder=holder)
    ranks.finish()
    check(exps[0], sets[0], "chunked")
    quads = sum((c1 - c0) * per_ct // 4 for c0, c1 in chunks)
    steps = ranks.take_stats()
    if holder >= 0:
        assert steps[holder] == 0
    assert sum(steps) == (quads * world if algo == "one_shot" else quads)

    src = [[x.cuda() for x in s] for s in sets]
    torch.cuda.synchronize()
    for k in range(20):
        for r in range(world):
            with torch.cuda.stream(ranks.streams[r]):
                ranks.bufs[r][lo:hi].copy_(src[k % 2][r])
            ranks.launch(r, algo, ctx, logn, hi - lo, blocks, threads, off=lo, holder=holder)
    ranks.finish()
    check(exps[1], sets[1], "20 launches back to back")


# ---------------------------------------------------------------------------------------------- (e)
def test_fused_transport_at_the_medical_cnn_size(monkeypatch):
    """109 ciphertexts of n = 4096 with 3 primes, 8 ranks, key holder 0: whole, then in the pipeline's chunks of
    20 ciphertexts through allreduce(view). The pipeline's 24-CTA all-reduce grid does not fit 8 ranks on one
    GPU, so the transports get the co-residency budget's grid instead."""
    monkeypatch.delenv("HEFL_ALLREDUCE_ALGO", raising=False)
    world, holder, n_ct = 8, 0, 109
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    L, n = ctx.L, ctx.n
    per_ct = 2 * L * n
    numel = n_ct * per_ct
    ts = make_transports(ctx, world, numel, holder)
    assert ts[0].pick_blocks(numel, "two_shot") * world <= cta_budget()
    qw = q_of_word(ctx.primes, numel, ctx.logn)
    gen = torch.Generator().manual_seed(109)
    inputs = [residues(qw, gen) for _ in range(world)]
    exp = ref_sum(inputs, qw)
    streams = [torch.cuda.Stream() for _ in ts]
    for chunks in ([(0, n_ct)], [(c0, min(n_ct, c0 + 20)) for c0 in range(0, n_ct, 20)]):
        for t, x in zip(ts, inputs):
            t.sym.tensor[:numel].copy_(x)
        torch.cuda.synchronize()
        transport_round(ts, streams, chunks, per_ct, (2, L, n))
        for r, t in enumerate(ts):
            assert t.last_algo == "two_shot"
            assert_words(t.sym.tensor[:numel], exp, f"{len(chunks)} chunk(s): rank {r}")
        steps = [t.peer_load_steps() for t in ts]
        want = [0] * world
        for c0, c1 in chunks:
            for r, (lo, hi) in enumerate(owner_ranges((c1 - c0) * per_ct // 4, world, holder)):
                want[r] += hi - lo
        assert steps[holder] == 0 and steps == want, (steps, want)


# ---------------------------------------------------------------------------------------------- (f)
@pytest.mark.parametrize("bits", [36, 61])
def test_pairwise_mask_gpu_matches_the_host_twin(bits):
    logn = 10
    gen = torch.Generator().manual_seed(bits)
    for L in range(1, 6):
        ctx = _ctx(logn, bits, L)
        numel = 3 * 2 * L << logn
        qw = q_of_word(ctx.primes, numel, logn)
        x = residues(qw, gen)
        for npeers in range(8):
            me, peers = 3, [2, 4, 1, 5, 0, 6, 7][:npeers]      # rank 3 of 8: peers below and above alternate
            seeds = [pair_seed(me, j) for j in peers]
            signs = [1 if j > me else -1 for j in peers]
            assert npeers < 2 or (1 in signs and -1 in signs)
            for rnd in (7, 0xFFFFFFFF):
                host = x.clone()
                ops.pairwise_mask_(host, seeds, signs, rnd, L, logn, ctx.consts_cpu)
                dev = x.cuda()
                ops.pairwise_mask_(dev, seeds, signs, rnd, L, logn, ctx.consts_cpu)
                what = f"{bits}-bit L={L} npeers={npeers} round={rnd:#x}"
                assert_words(dev, host, what)
                assert bool((host >= 0).all() and (host < qw).all()), what
                if npeers == 0:
                    assert torch.equal(host, x)


def test_pairwise_mask_grid_stride_at_the_medical_cnn_size():
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, enforce_security=False)
    numel = 109 * 2 * 3 * 4096
    assert numel // 2 > 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256   # several strides
    qw = q_of_word(ctx.primes, numel, ctx.logn)
    x = residues(qw, torch.Generator().manual_seed(3))
    seeds = [pair_seed(3, j) for j in (0, 1, 2, 4, 5, 6, 7)]
    signs = [-1, -1, -1, 1, 1, 1, 1]
    host = x.clone()
    ops.pairwise_mask_(host, seeds, signs, 0xFFFFFFFF, ctx.L, ctx.logn, ctx.consts_cpu)
    dev = x.cuda()
    ops.pairwise_mask_(dev, seeds, signs, 0xFFFFFFFF, ctx.L, ctx.logn, ctx.consts_cpu)
    assert_words(dev, host, "109 ciphertexts")


@pytest.mark.parametrize("world,holder,bits", [(2, -1, 61), (5, 0, 36), (8, 0, 61), (8, -1, 36)])
def test_masked_ranks_all_reduce_to_the_unmasked_sum(world, holder, bits):
    """The runner's rule: + towards higher ranks, - towards lower, round key round * 4096 + chunk."""
    logn, L = 12, 3
    ctx = _ctx(logn, bits, L)
    numel = 3 * 2 * L << logn
    qw = q_of_word(ctx.primes, numel, logn)
    gen = torch.Generator().manual_seed(world)
    inputs = [residues(qw, gen) for _ in range(world)]
    blocks = grid(world, 0)
    ranks = Ranks(world, numel, blocks)
    ranks.load(inputs)
    key = (5 * 4096 + 2) & 0xFFFFFFFF
    for r in range(world):
        peers = [j for j in range(world) if j != r]
        ops.pairwise_mask_(ranks.bufs[r], [pair_seed(r, j) for j in peers], [1 if j > r else -1 for j in peers],
                           key, L, logn, ctx.consts_cpu)
    torch.cuda.synchronize()
    if world > 1:
        for r in range(world):
            changed = (ranks.bufs[r].cpu() != inputs[r]).double().mean().item()
            assert changed > 0.99, f"rank {r}: only {changed:.4f} of the words are masked"
    ranks.run("two_shot", ctx, logn, numel, blocks, 512, holder=holder)
    exp = ref_sum(inputs, qw)
    for r in range(world):
        assert_words(ranks.bufs[r], exp, f"rank {r}")


# ---------------------------------------------------------------------------------------------- (g)
@pytest.mark.parametrize("K", [1, 7, 8, 9, 16, 17])
def test_local_sum_modq_of_many_maximal_addends(K):
    """Under a 61-bit prime 8 (q - 1) just fits in 64 bits and 9 (q - 1) does not, so a reduced accumulator may
    take 7 more addends, not 8. K = 16 and 17 are where reducing after every 8 addends would overflow."""
    logn, L = 12, 3
    ctx = _ctx(logn, 61, L)
    numel = 2 * 2 * L << logn
    qw = q_of_word(ctx.primes, numel, logn)
    gen = torch.Generator().manual_seed(K)
    for name, srcs in (("q - 1", [qw - 1] * K), ("random", [residues(qw, gen) for _ in range(K)])):
        exp = ref_sum(srcs, qw)
        out = torch.empty(numel, dtype=torch.int64, device="cuda")
        ops.local_sum_modq([s.cuda() for s in srcs], out, L, logn, ctx.consts.cuda())
        assert_words(out, exp, f"K={K} {name}: GPU")
        host = torch.empty(numel, dtype=torch.int64)
        ops.local_sum_modq(srcs, host, L, logn, ctx.consts)
        assert_words(host, exp, f"K={K} {name}: host twin")
