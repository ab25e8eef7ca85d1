"""GPU tests: every sm_90a HE kernel against its host C++ twin (bit-exact for integer
kernels) and the CKKS pipeline end to end. Run on an H100: pytest -m gpu."""
import pytest
import torch

from hefl_b200 import _ext
from hefl_b200.he.context import CKKSContext

pytestmark = pytest.mark.gpu
ops = _ext.ops()


def _ctx_pair(n, bits, scale_bits=40):
    c = CKKSContext(n, prime_bits=bits, scale_bits=scale_bits, enforce_security=False)
    g = CKKSContext(n, primes=c.primes, scale_bits=scale_bits, enforce_security=False, device="cuda")
    return c, g


@pytest.mark.parametrize("logn,bits", [(10, (27,)), (11, (54,)), (12, (36, 36, 37)), (12, (54, 55)), (12, (58, 57)),
                                       (13, (54, 54, 54, 55)), (13, (40,) * 8), (14, (54, 54, 54, 54)),
                                       (14, (60, 59, 58)), (15, (60, 60))])
def test_ntt_gpu_matches_cpu(logn, bits):
    n = 1 << logn
    c, g = _ctx_pair(n, bits)
    L = len(bits)
    gen = torch.Generator().manual_seed(logn)
    a = torch.stack([torch.randint(0, q, (5, n), generator=gen, dtype=torch.int64) for q in c.primes], dim=1).contiguous()
    ref = a.clone()
    ops.ntt_(ref, c.tables, c.consts, L, logn, False)
    x = a.cuda()
    ops.ntt_(x, g.tables, g.consts, L, logn, False)
    assert torch.equal(x.cpu(), ref)
    ops.ntt_(x, g.tables, g.consts, L, logn, True)
    assert torch.equal(x.cpu(), a)


def test_pointwise_and_reduce_gpu_match_cpu():
    c, g = _ctx_pair(4096, (36, 36, 37))
    gen = torch.Generator().manual_seed(0)
    a = torch.stack([torch.randint(0, q, (4, 2, 4096), generator=gen, dtype=torch.int64) for q in c.primes], dim=2).contiguous()
    b = torch.stack([torch.randint(0, q, (2, 4096), generator=gen, dtype=torch.int64) for q in c.primes], dim=1).contiguous()
    for op in (0, 1, 2, 3):
        ref = a.clone()
        ops.pointwise_(ref, a, b, 3, c.consts, op)
        out = a.clone().cuda()
        ops.pointwise_(out, a.cuda(), b.cuda(), 3, g.consts, op)
        assert torch.equal(out.cpu(), ref), op
    big = torch.randint(-2**63, 2**63 - 1, (6, 4096), generator=gen, dtype=torch.int64)
    ref = big.clone()
    ops.reduce_mod_(ref, 3, c.consts)
    out = big.cuda()
    ops.reduce_mod_(out, 3, g.consts)
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("n,bits", [(1024, (27,)), (2048, (54,)), (4096, (36, 36, 37)), (4096, (58, 50)),
                                    (8192, (54, 54, 54, 55)), (16384, (54, 54, 54, 54)), (32768, (60, 60))])
def test_encrypt_decrypt_gpu_bit_exact_vs_cpu(n, bits):
    c, g = _ctx_pair(n, bits)
    sk, pk = c.keygen(seed=5)
    gen = torch.Generator().manual_seed(1)
    vals = torch.randn(n + 100, generator=gen)
    msg = c.encode(vals)
    msg_g = g.encode(vals.cuda())
    assert (msg_g.cpu() - msg).abs().max() <= 1  # fp64 FFT: rounding may differ by one unit
    L = len(bits)
    ct_c = ops.encrypt(msg, pk, msg.shape[0], L, c.logn, c.tables, c.consts, None, 77, 3)
    ct_g = ops.encrypt(msg.cuda(), pk.cuda(), msg.shape[0], L, g.logn, g.tables, g.consts, None, 77, 3)
    assert torch.equal(ct_g.cpu(), ct_c)
    res_c = ops.decrypt(ct_c, sk, min(L, 2), c.logn, c.tables, c.consts)
    res_g = ops.decrypt(ct_g, sk.cuda(), min(L, 2), g.logn, g.tables, g.consts)
    assert torch.equal(res_g.cpu(), res_c)
    cc = ops.crt_center(res_c, c.consts_cpu, c.q0_inv_q1)
    cg = ops.crt_center(res_g, g.consts_cpu, g.q0_inv_q1)
    assert torch.equal(cg.cpu(), cc)


def test_fedavg_end_to_end_on_gpu():
    g = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    sk, pk = g.keygen(seed=9)
    gen = torch.Generator().manual_seed(2)
    K = 8
    ws = [torch.randn(222722, generator=gen).cuda() * 0.05 for _ in range(K)]
    cts = [g.encrypt(w, pk, seed=10 + i) for i, w in enumerate(ws)]
    assert cts[0].count == 109
    agg = g.sum_batches(cts)
    out = g.decrypt(agg, sk, divide_by=K)
    ref = torch.stack(ws).mean(0)
    assert out.shape == ref.shape
    assert (out - ref).abs().max() < 1e-6


def test_coeff_packing_and_scalar_mul_gpu():
    g = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    sk, pk = g.keygen(seed=4)
    vals = torch.linspace(-2, 2, 6000).cuda()
    ct = g.encrypt(vals, pk, seed=9, packing="coeff")
    out = g.decrypt(ct, sk)
    assert (out - vals).abs().max() < 1e-6
    ct2 = g.encrypt(vals[:2048], pk, seed=10)
    g.mul_scalar_(ct2, 0.125)
    assert (g.decrypt(ct2, sk) - vals[:2048] * 0.125).abs().max() < 1e-4


def test_ct_ct_multiply_gpu():
    g = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    sk, pk = g.keygen(seed=8)
    rlk = g.relin_keygen(sk, seed=8, digit_bits=12)
    a = torch.linspace(-1, 1, 2048).cuda()
    b = torch.linspace(0.5, 1.5, 2048).cuda()
    prod = g.multiply(g.encrypt(a, pk, seed=14), g.encrypt(b, pk, seed=15), rlk)
    assert (g.decrypt(prod, sk) - a * b).abs().max() < 5e-3


def test_local_sum_modq_gpu_matches_cpu():
    c, g = _ctx_pair(4096, (36, 36, 37))
    gen = torch.Generator().manual_seed(3)
    srcs = [torch.stack([torch.randint(0, q, (3, 2, 4096), generator=gen, dtype=torch.int64) for q in c.primes], dim=2).contiguous()
            for _ in range(5)]
    ref = torch.empty_like(srcs[0])
    ops.local_sum_modq(srcs, ref, 3, 12, c.consts)
    exp = sum(s.clone() for s in srcs)
    for l, q in enumerate(c.primes):
        assert torch.equal(ref[:, :, l], exp[:, :, l] % q)
    out = torch.empty_like(srcs[0]).cuda()
    ops.local_sum_modq([s.cuda() for s in srcs], out, 3, 12, g.consts)
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("world,algo", [(1, 0), (1, 1), (2, 0), (2, 1), (4, 0), (4, 1)])
def test_fused_allreduce_protocol_single_gpu(world, algo):
    """The multi-rank flag protocol exercised on ONE GPU: `world` logical ranks with their own
    buffers and signal pads run the kernel concurrently on separate streams."""
    c, g = _ctx_pair(4096, (36, 36, 37))
    gen = torch.Generator().manual_seed(world * 10 + algo)
    shape = (7, 2, 3, 4096)
    numel = 7 * 2 * 3 * 4096
    inputs = [torch.stack([torch.randint(0, q, (7, 2, 4096), generator=gen, dtype=torch.int64) for q in c.primes], dim=2).contiguous()
              for _ in range(world)]
    exp = sum(x.clone() for x in inputs)
    for l, q in enumerate(c.primes):
        exp[:, :, l] %= q
    bufs = [x.cuda().reshape(-1).clone() for x in inputs]
    blocks = 4
    sigs = [torch.zeros(2 * blocks * world + 64, dtype=torch.int32, device="cuda") for _ in range(world)]
    outs = [torch.zeros(numel, dtype=torch.int64, device="cuda") for _ in range(world)]
    status = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    torch.cuda.synchronize()
    for r in range(world):
        with torch.cuda.stream(streams[r]):
            ops.allreduce_modq([b.data_ptr() for b in bufs], [s.data_ptr() for s in sigs], 0,
                               outs[r] if algo == 1 else None, status[r], g.consts_cpu, numel, 3, 12,
                               r, world, algo, blocks, 256, 3000)
    torch.cuda.synchronize()
    for r in range(world):
        assert int(status[r].item()) == 0
        got = (outs[r] if algo == 1 else bufs[r]).view(shape).cpu()
        assert torch.equal(got, exp), (r, algo)
        assert int(sigs[r].abs().sum().item()) == 0  # flags returned to rest


def test_fused_allreduce_timeout_is_detected():
    """Fault injection: a 2-rank launch where rank 1 never shows up must time out, not hang."""
    c, g = _ctx_pair(4096, (36,))
    numel = 2 * 4096
    buf = torch.zeros(numel, dtype=torch.int64, device="cuda")
    sig = torch.zeros(256, dtype=torch.int32, device="cuda")
    sig_peer = torch.ones(256, dtype=torch.int32, device="cuda")  # peer pad never drains
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.allreduce_modq([buf.data_ptr(), buf.data_ptr()], [sig.data_ptr(), sig_peer.data_ptr()], 0, None,
                       status, g.consts_cpu, numel, 1, 12, 0, 2, 0, 2, 64, 50)
    torch.cuda.synchronize()
    assert int(status.item()) != 0


def test_pipelined_fedavg_matches_unchunked():
    """Chunked 3-stream encrypt / all-reduce / decrypt pipeline == the single-shot path."""
    from hefl_b200.config import FLConfig
    from hefl_b200.fl import FederatedRunner

    cfg = FLConfig(model="medcnn", local_epochs=1, steps_per_epoch=1, val_steps=0, nn_backend="cudnn",
                   transport="fused", device="cuda")
    run = FederatedRunner(cfg, device=torch.device("cuda"))
    w = run.pack.flat.clone()
    run.fedavg_pipelined(chunk_cts=20)
    torch.cuda.synchronize()
    assert (run.pack.flat - w).abs().max() < 1e-6        # one client: average == its own weights
    run.pack.load_flat(w)
    ct = run.encrypt_update()
    agg = run.aggregate(ct)
    run.decrypt_apply(agg)
    assert (run.pack.flat - w).abs().max() < 1e-6


@pytest.mark.parametrize("n,bits", [(2048, (54, 50)), (4096, (36, 36, 37)), (8192, (54, 54, 54, 55))])
def test_fused_rescale_and_keyswitch_match_the_reference_loops(n, bits):
    """The one-launch rescale and key-switch kernels (he_eval2.cu) against the limb-by-limb reference path that
    runs on the host twin: exact modular arithmetic, so the ciphertexts must be identical word for word."""
    from hefl_b200.he.context import CtBatch, RelinKey

    c, g = _ctx_pair(n, bits)
    sk, pk = c.keygen(seed=3)
    rlk_c = c.relin_keygen(sk, seed=4, digit_bits=14)
    rlk_g = RelinKey([k.cuda() for k in rlk_c.keys], rlk_c.digit_bits)
    gen = torch.Generator().manual_seed(5)
    nv = 3 * (n // 2) - 7                                  # three ciphertexts: a partial unit for n < 8192
    va, vb = torch.rand(nv, generator=gen) * 2 - 1, torch.rand(nv, generator=gen) + 0.5
    ca, cb = c.encrypt(va, pk, seed=1), c.encrypt(vb, pk, seed=2)
    ga = CtBatch(ca.data.cuda(), ca.scale, ca.nvals, ca.packing)
    gb = CtBatch(cb.data.cuda(), cb.scale, cb.nvals, cb.packing)
    # rescale alone (after a scalar multiply) ...
    r_c = c.mul_scalar_(ca.clone(), 0.375)
    r_g = g.mul_scalar_(ga.clone(), 0.375)
    assert r_g.level == len(bits) - 1 and torch.equal(r_g.data.cpu(), r_c.data)
    # ... and the whole ct x ct path: tensor product, key switch, rescale
    p_c = c.multiply(ca, cb, rlk_c, rescale=True)
    p_g = g.multiply(ga, gb, rlk_g, rescale=True)
    assert torch.equal(p_g.data.cpu(), p_c.data)
    out = g.decrypt(p_g, sk.cuda())
    assert (out.cpu() - va * vb).abs().max() < 5e-3


@pytest.mark.parametrize("n,bits", [(2048, (54, 50)), (4096, (36, 36, 37)), (8192, (54, 54, 54, 55))])
def test_device_key_generation_is_bit_identical_to_the_host_twin(n, bits):
    """Secret key, public key and the digit-decomposed evaluation keys generated by the CUDA kernels (same Philox
    streams, batched NTT) against the host C++ twin, which the CPU suite ties to the big-integer oracle."""
    c, g = _ctx_pair(n, bits)
    sk_c, pk_c = c.keygen(seed=21)
    sk_g, pk_g = g.keygen(seed=21)
    assert sk_g.is_cuda and pk_g.is_cuda
    assert torch.equal(sk_g.cpu(), sk_c) and torch.equal(pk_g.cpu(), pk_c)
    r_c = c.relin_keygen(sk_c, seed=22, digit_bits=13)
    r_g = g.relin_keygen(sk_g, seed=22, digit_bits=13)
    assert len(r_c.keys) == len(r_g.keys) == len(bits)
    for kc, kg in zip(r_c.keys, r_g.keys):
        assert kg.is_cuda and torch.equal(kg.cpu(), kc)
    # and the keys work: encrypt under the device pk, multiply, relinearise with the device evk, decrypt
    vals = torch.linspace(-1, 1, n // 2, device="cuda")
    ct = g.encrypt(vals, pk_g, seed=5)
    prod = g.multiply(ct, ct, r_g)
    back = g.decrypt(prod, sk_g)
    assert float((back[: n // 2] - vals * vals).abs().max()) < 1e-3
