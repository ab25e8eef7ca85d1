"""The persistent sm_90a HE kernels where the dispatcher actually selects them, and the CKKS decode against a
reference that shares nothing with the library.

`ntt2_kernel`, `encrypt2_kernel` and `decrypt2_kernel` are persistent: one CTA per SM, clusters of two CTAs dealt
round-robin to the RNS limbs, each CTA looping over units of 8192 coefficients. Their interesting paths (the
load/store ring wrapping, tail units, unequal cluster counts per limb, SM budgets, the N = 16384 scratch rows) only
run at batch sizes several times the number of workers. The sizes below are derived from the SM count and the CTA
budget; every GPU test then asks torch.profiler which kernels ran, so the coverage is checked, not assumed. Integer
results must equal the host C++ twin (`ops.*` on CPU tensors) word for word.

The decode reference is exact CRT centring with Python integers followed by a plain float64 FFT of length 2N: slot j
of m is m(zeta^(5^j)) with zeta = exp(i*pi/N), i.e. 2N * ifft(pad(m, 2N))[5^j mod 2N]. The CPU tests tie it to
`oracle.ckks_slots_of` and to the host twin; the GPU tests compare the fused decode kernel with both."""
import contextlib

import numpy as np
import pytest
import torch

from hefl_b200 import _ext
from hefl_b200.he import oracle
from hefl_b200.he.bfv import BFVFracContext, BFVRelinKey
from hefl_b200.he.context import CKKSContext, CtBatch
from kernel_trace import kernels_run, ran

ops = _ext.ops()
gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- helpers
@pytest.fixture
def cta_budget():
    """`with cta_budget(ntt, enc, dec):` sets the persistent kernels' per-role CTA budgets and restores the whole chip
    on exit; the fixture restores it once more at teardown, so no test leaves a budget behind."""

    @contextlib.contextmanager
    def budget(ntt, enc, dec):
        ops.set_he_cta_limits(ntt, enc, dec)
        try:
            yield
        finally:
            ops.set_he_cta_limits(0, 0, 0)

    yield budget
    ops.set_he_cta_limits(0, 0, 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _budget(name):
    """(ntt, encrypt, decrypt) CTA budgets: the whole chip, a tiny encrypt budget, and the split the pipelined
    FedAvg round uses on one node (all-reduce 24 SMs, decrypt 28, encrypt the rest)."""
    return {"chip": (0, 0, 0), "enc8": (0, 8, 0), "pipeline": (0, _sms() - 52, 28), "dec28": (0, 0, 28)}[name]


def _grid(limit=0):
    """CTAs of a persistent launch: an even number (clusters of two), one per SM or the budget."""
    g = _sms() & ~1
    if 0 < limit < g:
        g = limit & ~1
    return max(g, 2)


def _max_workers(grid, limbs):
    """CTAs of the busiest limb: the grid's clusters are dealt round-robin to the limbs."""
    return 2 * -(-(grid // 2) // limbs)


def _polys(logn):
    """Polynomials per unit of work: 8192 coefficients, at least one polynomial."""
    return max(1, 8192 >> logn)


def _count(units, logn):
    """A batch of `units` units whose last unit is partial (one polynomial short) wherever a unit holds several;
    odd either way."""
    p = _polys(logn)
    return units * p - 1 if p > 1 else units | 1


def _ctx_pair(n, bits, scale_bits=40):
    c = CKKSContext(n, prime_bits=bits, scale_bits=scale_bits, enforce_security=False)
    g = CKKSContext(n, primes=c.primes, scale_bits=scale_bits, enforce_security=False, device="cuda")
    return c, g


def _residues(primes, lead, n, gen):
    """Uniform residues [*lead, L, N], limb l below primes[l]."""
    return torch.stack([torch.randint(0, q, (*lead, n), generator=gen, dtype=torch.int64) for q in primes],
                       dim=-2).contiguous()


def assert_same_words(got, want):
    got = got.cpu()
    assert got.shape == want.shape, (tuple(got.shape), tuple(want.shape))
    if torch.equal(got, want):
        return
    bad = (got != want).nonzero()
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{bad.shape[0]} of {want.numel()} words differ; first at {i}: "
                         f"{int(got[i])} != {int(want[i])}")


# ---------------------------------------------------------------------------------------------- decode reference
def crt_centered(res, primes):
    """Exact centred CRT lift (-Q/2, Q/2] of residues [..., k, N] (int64): `oracle.crt_centered`, vectorised over
    Python integers."""
    Q = 1
    for q in primes:
        Q *= q
    x = 0
    for l, q in enumerate(primes):
        Qi = Q // q
        x = x + res[..., l, :].astype(object) * (Qi * pow(Qi, -1, q))
    x = x % Q
    return np.where(x > Q // 2, x - Q, x)


def _slot_index(n):
    return np.array([pow(5, j, 2 * n) for j in range(n // 2)])


def slots_of(coeffs):
    """Complex slots [C, N/2] of real polynomials coeffs [C, N]: slot j = m(zeta^(5^j)), zeta = exp(i*pi/N)."""
    coeffs = np.asarray(coeffs, dtype=np.float64)
    n = coeffs.shape[-1]
    z = 2 * n * np.fft.ifft(np.pad(coeffs, ((0, 0), (0, n))), axis=1)
    return z[:, _slot_index(n)]


def coeffs_of_slots(z, n):
    """Real coefficients [C, N] (float64) of the polynomials whose slots are the real values z [C, N/2]: the
    inverse of `slots_of` (the value at zeta^g and its conjugate at zeta^-g, one length-2N FFT)."""
    g = _slot_index(n)
    X = np.zeros((z.shape[0], 2 * n), dtype=np.complex128)
    X[:, g] = z
    X[:, (-g) % (2 * n)] = z
    return (np.fft.fft(X, axis=1)[:, :n] / n).real


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def assert_within_f32(got, want, ulps=1):
    """|got - want| <= ulps float32 spacings of want, plus 1e-12 of the largest |want| for values that are zero up to
    cancellation in a float64 FFT."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    err = np.abs(got - want)
    tol = ulps * ulp32(want) + 1e-12 * np.abs(want).max()
    bad = np.nonzero(err > tol)[0]
    assert bad.size == 0, (f"{bad.size} of {want.size} values off; first at {bad[0]}: {got[bad[0]]!r} vs "
                           f"{want[bad[0]]!r} (tolerance {tol[bad[0]]:.3g})")


def wrap_edges(Q):
    """Integers at both sides of the centring decision: +-floor(Q/2) and their neighbours, 0 and -1."""
    h = Q // 2
    return [h, -h, h - 1, -h + 1, h - 2**40, -h + 2**40, 0, -1]


K_CLIENTS = 3


def decode_case(logn, k, seed=0):
    """Decrypted residues of three ciphertexts (two with slots whose Delta*K*|v| lies within 1 % of
    max_abs_message(k), both signs, mixed with ordinary values; one with uniform residues and the wrap edges) plus
    their exact centred coefficients. Returns (cpu context, res [3, k, N] int64, coeffs [3, N] object, inv_scale,
    nvals ending mid-ciphertext)."""
    n = 1 << logn
    c = CKKSContext(n, prime_bits=(54, 50), scale_bits=40, enforce_security=False)
    primes = c.primes[:k]
    Q = 1
    for q in primes:
        Q *= q
    M = c.max_abs_message(k)
    rng = np.random.default_rng(1000 * logn + k + seed)
    z = rng.standard_normal((2, n // 2)) * (M / 8)
    edge = rng.uniform(0.99, 1.0, (2, n // 4)) * M
    edge[:, 1::2] *= -1
    z[:, ::2] = edge
    base = coeffs_of_slots(z, n)
    rows = [[int(t) + int(e) for t, e in zip(row, rng.integers(-2**20, 2**20, n))] for row in base]
    wild = [int(rng.integers(0, 2**62)) * 2**62 % Q + int(rng.integers(0, 2**62)) for _ in range(n)]
    wild = [((w % Q) + Q // 2) % Q - Q // 2 for w in wild]
    wild[: len(wrap_edges(Q))] = wrap_edges(Q)
    coeffs = np.array(rows + [wild], dtype=object)
    res = np.stack([np.stack([np.array([int(v % q) for v in row], dtype=np.int64) for q in primes])
                    for row in coeffs])
    inv = 1.0 / (c.scale * K_CLIENTS)
    nvals = 3 * n // 2 - n // 4 - 3
    return c, torch.from_numpy(res), coeffs, inv, nvals


def reference_decode(coeffs, inv, nvals):
    """float64 decode of exact coefficients: centred integer -> float64 (correctly rounded) -> slots -> * inv."""
    return (slots_of(np.array(coeffs, dtype=np.float64)).real * inv).reshape(-1)[:nvals]


# ---------------------------------------------------------------------------------------------- CPU: the reference
def test_slot_reference_is_the_canonical_embedding():
    n = 64
    rng = np.random.default_rng(3)
    m = rng.integers(-2**30, 2**30, (2, n)).astype(np.float64)
    got = slots_of(m)
    for row, zrow in zip(m, got):
        want = np.array(oracle.ckks_slots_of(list(row), n))
        assert np.abs(zrow - want).max() <= 1e-9 * np.abs(want).max()
    v = rng.standard_normal((2, n // 2))
    back = slots_of(coeffs_of_slots(v, n))
    assert np.abs(back.real - v).max() < 1e-12 and np.abs(back.imag).max() < 1e-12


def test_crt_reference_matches_the_oracle_at_the_wrap():
    c = CKKSContext(1024, prime_bits=(54, 50), scale_bits=40, enforce_security=False)
    Q = c.primes[0] * c.primes[1]
    xs = wrap_edges(Q) + [Q // 4, -(Q // 4), 12345, -12345]
    res = np.array([[[x % q for x in xs] for q in c.primes]], dtype=np.int64)
    got = crt_centered(res, c.primes)[0]
    assert list(got) == xs
    assert [oracle.crt_centered([x % q for q in c.primes], c.primes) for x in xs] == xs


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("logn", [10, 11, 12, 13, 14, 15])
def test_host_decode_matches_the_slot_reference(logn, k):
    c, res, coeffs, inv, nvals = decode_case(logn, k)
    assert (crt_centered(res.numpy(), c.primes[:k]) == coeffs).all()
    host = ops.ckks_decode_residues(res, c.consts_cpu, c.q0_inv_q1, logn, inv, c.rot, c.ksi, nvals)
    assert host.shape == (nvals,)
    assert_within_f32(host.numpy(), reference_decode(coeffs, inv, nvals))
    # the host centring, at the wrap and over the edge band, against the exact integers
    cc = ops.crt_center(res, c.consts_cpu, c.q0_inv_q1).numpy()
    exact = np.array(coeffs, dtype=np.float64)
    assert (np.abs(cc - exact) <= np.abs(exact) * 2.0**-52).all()


@pytest.mark.parametrize("logn", [10, 12, 15])
def test_host_encode_is_within_half_n_of_the_scaled_slots(logn):
    n = 1 << logn
    c = CKKSContext(n, prime_bits=(54,), scale_bits=40, enforce_security=False)
    v = torch.randn(n + 77, generator=torch.Generator().manual_seed(logn), dtype=torch.float64)
    w = 1.37
    msg = c.encode(v, scale=c.scale * w)
    _check_encode(msg, v, c.scale * w)


def _check_encode(msg, v, scale):
    """Every slot of the integer message is within N/2 of scale * v: each coefficient is rounded by at most 1/2."""
    n = msg.shape[-1]
    z = slots_of(msg.cpu().numpy().astype(np.float64)).reshape(-1)
    want = np.zeros(z.size)
    want[: v.numel()] = v.double().cpu().numpy() * scale
    tol = n / 2 + 1e-12 * np.abs(want).max()
    assert np.abs(z.real - want).max() <= tol
    assert np.abs(z.imag).max() <= tol


# ---------------------------------------------------------------------------------------------- 1. NTT ring
# bits -> the inverse correction schedule pick_corr selects: none, before pass 1, before every pass but the first
NTT_CASES = [(logn, bits, corr) for logn in (10, 11, 12, 13, 14)
             for bits, corr in ((40, 0), (53, 2), (56, 3 if logn <= 12 else 7))]


@gpu
@pytest.mark.parametrize("logn,bits,corr", NTT_CASES)
def test_ntt2_ring_wraps_with_partial_units_and_unequal_limbs(logn, bits, corr, cta_budget):
    """Forward and inverse NTT of rows that give every worker at least three units (the ring's buffers are reused
    and the barrier parity flips), with a partial last unit, on four limbs: at full chip, and under a 10-CTA budget
    whose five clusters give the limbs 2, 1, 1, 1."""
    n = 1 << logn
    L = 4
    c, g = _ctx_pair(n, (bits,) * L)
    assert {p.bit_length() for p in c.primes} == {bits}
    gen = torch.Generator().manual_seed(100 * logn + bits)
    for limit in (0, 10):
        with cta_budget(limit, 0, 0):
            J = 3 * _max_workers(_grid(limit), L) * _polys(logn) + 1          # polynomials per limb
            a = _residues(c.primes, (J,), n, gen)
            ref = a.clone()
            ops.ntt_(ref, c.tables, c.consts, L, logn, False)
            a_g, ref_g = a.cuda(), ref.cuda()
            x = torch.empty_like(a_g)
            # each transform starts from a fresh copy of its input, so that kernels_run may repeat it
            _, fwd = kernels_run(lambda: ops.ntt_(x.copy_(a_g), g.tables, g.consts, L, logn, False))
            assert_same_words(x, ref)
            # the forward result is arbitrary residues; the inverse must return exactly a (= the host inverse of ref)
            _, inv = kernels_run(lambda: ops.ntt_(x.copy_(ref_g), g.tables, g.consts, L, logn, True))
            assert_same_words(x, a)
            assert ran(fwd, f"ntt2_kernel<{logn}, false, 0u>"), (limit, sorted(fwd))
            assert ran(inv, f"ntt2_kernel<{logn}, true, {corr}u>"), (limit, sorted(inv))


# ---------------------------------------------------------------------------------------------- 2. encrypt2
ENC_CASES = [(1024, (40,)), (2048, (54, 50)), (4096, (58, 50, 45)), (8192, (54, 54, 54, 55)),
             (16384, (54, 54, 54, 54))]


@gpu
@pytest.mark.parametrize("budget", ["chip", "enc8", "pipeline"])
@pytest.mark.parametrize("n,bits", ENC_CASES)
def test_encrypt2_matches_host_twin(n, bits, budget, cta_budget):
    """The persistent encrypt at a batch just above two units per worker (odd, partial last unit), with a message
    at a nonzero ciphertext offset and as an encryption of zero."""
    c, g = _ctx_pair(n, bits)
    L, logn = c.L, c.logn
    _, pk = c.keygen(seed=31)
    pk_g = pk.cuda()
    limits = _budget(budget)
    gen = torch.Generator().manual_seed(n + L)
    with cta_budget(*limits):
        C = _count(2 * _max_workers(_grid(limits[1]), L) + 1, logn)
        msg = torch.randint(-2**62, 2**62, (C, n), generator=gen, dtype=torch.int64)
        msg_g = msg.cuda()
        for m, m_g, seed, off in ((msg, msg_g, 41, 1000 + C), (None, None, 42, 0)):
            ref = ops.encrypt(m, pk, C, L, logn, c.tables, c.consts, None, seed, off)
            out, names = kernels_run(lambda: ops.encrypt(m_g, pk_g, C, L, logn, g.tables, g.consts, None, seed, off))
            assert ran(names, f"encrypt2_kernel<{logn}>"), (C, sorted(names))
            assert_same_words(out, ref)


# ---------------------------------------------------------------------------------------------- 3. chunked encrypt
@gpu
@pytest.mark.parametrize("kernel", ["encrypt_kernel", "encrypt2_kernel"])
def test_chunked_encrypt_into_one_buffer_equals_one_whole_call(kernel):
    """What the pipelined FedAvg round does: encrypt chunk by chunk into views of one buffer, with each chunk's
    ciphertext offset and the client's weight. The bytes must be those of one call on the whole vector."""
    g = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40, device="cuda")
    _, pk = g.keygen(seed=51)
    chunk = 20 if kernel == "encrypt_kernel" else _count(2 * _max_workers(_grid(), g.L) + 1, g.logn)
    n_ct = 2 * chunk + 7
    vals = torch.randn(n_ct * g.slots - 123, generator=torch.Generator().manual_seed(5)).cuda() * 0.05
    w = 1.37
    whole = g.encrypt(vals, pk, seed=77, weight=w)
    per = 2 * g.L * g.n
    buf = torch.zeros(n_ct * per, dtype=torch.int64, device="cuda")

    def chunks():
        for c0 in range(0, n_ct, chunk):
            c1 = min(n_ct, c0 + chunk)
            g.encrypt(vals[c0 * g.slots: c1 * g.slots], pk, seed=77, out=buf[c0 * per: c1 * per], ct_offset=c0,
                      weight=w)

    _, names = kernels_run(chunks)
    assert ran(names, kernel + "<"), sorted(names)
    if kernel == "encrypt_kernel":
        assert not ran(names, "encrypt2_kernel")
    assert_same_words(buf.view(n_ct, 2, g.L, g.n), whole.data.cpu())


# ---------------------------------------------------------------------------------------------- 4. decrypt2
DEC_CASES = [  # n, bits, k, rescaled first, budget
    (1024, (40, 40), 2, False, "chip"),
    (2048, (54, 50, 50), 2, True, "chip"),
    (4096, (36, 36, 37), 1, False, "chip"),
    (4096, (36, 36, 37), 2, False, "dec28"),
    (8192, (54, 54, 54, 55), 2, True, "chip"),
    (16384, (50, 50, 50), 2, False, "dec28"),
]


@gpu
@pytest.mark.parametrize("n,bits,k,rescaled,budget", DEC_CASES)
def test_decrypt2_with_many_units_per_worker(n, bits, k, rescaled, budget, cta_budget):
    """The fused decrypt over at least three units per worker and an odd batch (the tail of the last unit is clamped),
    for one and two limbs, and for a ciphertext one level down (fewer limbs than the tables)."""
    c, g = _ctx_pair(n, bits)
    logn = c.logn
    sk, _ = c.keygen(seed=61)
    limits = _budget(budget)
    gen = torch.Generator().manual_seed(n + k)
    with cta_budget(*limits):
        C = _count(3 * _max_workers(_grid(limits[2]), k) + 1, logn)
        ct = _residues(c.primes, (C, 2), n, gen)
        if rescaled:
            ct = c.rescale_(CtBatch(ct, c.scale * c.primes[-1], 0)).data
            assert ct.shape[2] == c.L - 1
        ref = ops.decrypt(ct, sk, k, logn, c.tables, c.consts)
        ct_g, sk_g = ct.cuda(), sk.cuda()
        out, names = kernels_run(lambda: ops.decrypt(ct_g, sk_g, k, logn, g.tables, g.consts))
    assert ran(names, f"decrypt2_kernel<{logn}, "), (C, sorted(names))
    assert_same_words(out, ref)


# ---------------------------------------------------------------------------------------------- 5. decode
@gpu
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("logn", [10, 11, 12, 13, 14, 15])
def test_decode_residues_matches_host_twin_and_slot_reference(logn, k):
    c, res, coeffs, inv, nvals = decode_case(logn, k)
    g = CKKSContext(c.n, primes=c.primes, scale_bits=40, enforce_security=False, device="cuda")
    res_g = res.cuda()
    out, names = kernels_run(lambda: ops.ckks_decode_residues(res_g, g.consts_cpu, g.q0_inv_q1, logn, inv, g.rot,
                                                              g.ksi, nvals))
    assert ran(names, "ckks_decode_res_kernel("), sorted(names)
    got = out.cpu().numpy()
    host = ops.ckks_decode_residues(res, c.consts_cpu, c.q0_inv_q1, logn, inv, c.rot, c.ksi, nvals).numpy()
    assert_within_f32(got, host)
    assert_within_f32(got, reference_decode(coeffs, inv, nvals))


@gpu
@pytest.mark.parametrize("k", [1, 2])
def test_crt_center_at_the_wrap_against_big_integers(k):
    c, res, coeffs, _, _ = decode_case(12, k, seed=1)
    g = CKKSContext(c.n, primes=c.primes, scale_bits=40, enforce_security=False, device="cuda")
    # the kernel converts the 128-bit magnitude as hi * 2^64 + lo, the host twin in one rounding: both stay within
    # one rounding of the exact integer, not necessarily on the same side
    got = ops.crt_center(res.cuda(), g.consts_cpu, g.q0_inv_q1).cpu()
    exact = np.array(coeffs, dtype=np.float64)
    err = np.abs(got.numpy() - exact)
    assert (err <= np.abs(exact) * 2.0**-52).all()
    Q = c.primes[0] * (c.primes[1] if k == 2 else 1)
    edges = np.array(wrap_edges(Q), dtype=np.float64)
    assert (np.sign(got.numpy()[2, : edges.size]) == np.sign(edges)).all()


@gpu
@pytest.mark.parametrize("logn", [10, 11, 12, 13, 14, 15])
def test_gpu_encode_is_within_half_n_of_the_scaled_slots(logn):
    n = 1 << logn
    c, g = _ctx_pair(n, (54,))
    v = torch.randn(2 * n + 77, generator=torch.Generator().manual_seed(logn), dtype=torch.float32)
    for w in (1.0, 0.37, 2.5):
        msg_g, names = kernels_run(lambda: g.encode(v.cuda(), scale=g.scale * w))
        assert ran(names, "ckks_encode_kernel("), sorted(names)
        assert (msg_g.cpu() - c.encode(v, scale=c.scale * w)).abs().max() <= 1
        _check_encode(msg_g, v, g.scale * w)


# ---------------------------------------------------------------------------------------------- 6. BFV on CUDA
def _bfv_pair():
    cpu = BFVFracContext(p=65537, m=2048, sec=128)
    return cpu, BFVFracContext(p=65537, m=2048, sec=128, q=cpu.q, device="cuda")


@gpu
def test_bfv_fractional_codec_on_cuda_matches_the_oracle():
    cpu, dev = _bfv_pair()
    vals = [0.0, 1.0, -1.0, 0.5, -0.375, 3.1415926, -123.456, 1e-5, 2**20 + 0.25, -(2.0**40) - 2.0**-30,
            2.0**63, -(2.0**-32), 0.999999999]
    vals += torch.randn(19, generator=torch.Generator().manual_seed(7), dtype=torch.float64).mul(1e3).tolist()
    v = torch.tensor(vals, dtype=torch.float64)
    msg = dev.encode(v.cuda())
    assert torch.equal(msg.cpu(), cpu.encode(v))
    for x, row in zip(vals, msg.cpu().tolist()):
        assert row == oracle.frac_encode(x, dev.n)
    back = dev.decode(msg).cpu()
    assert torch.equal(back, cpu.decode(msg.cpu()))
    assert back.tolist() == [oracle.frac_decode(r) for r in msg.cpu().tolist()]


@gpu
@pytest.mark.parametrize("size", ["small", "persistent"])
def test_bfv_encrypt_with_delta_scale_and_decrypt_on_cuda(size):
    """BFV encrypts with msg_scale = Delta (one ciphertext per scalar, one 54-bit limb): a few scalars on the
    one-CTA-per-ciphertext kernel, and a batch large enough for the persistent one."""
    cpu, dev = _bfv_pair()
    sk, pk = cpu.keygen(seed=71)
    C = 9 if size == "small" else _count(2 * _max_workers(_grid(), 1) + 1, dev.logn)
    vals = torch.randn(C, generator=torch.Generator().manual_seed(C), dtype=torch.float64) * 100
    ref = cpu.encrypt(vals, pk, seed=72, ct_offset=5)
    out, names = kernels_run(lambda: dev.encrypt(vals.cuda(), pk.cuda(), seed=72, ct_offset=5))
    if size == "small":
        assert ran(names, "encrypt_kernel<") and not ran(names, "encrypt2_kernel"), sorted(names)
    else:
        assert ran(names, f"encrypt2_kernel<{dev.logn}>"), (C, sorted(names))
    assert_same_words(out, ref)
    digits, names = kernels_run(lambda: dev.decrypt_digits(out, sk.cuda()))
    assert ran(names, f"decrypt2_kernel<{dev.logn}, ") and ran(names, "bfv_scale_round_kernel("), sorted(names)
    assert_same_words(digits, cpu.decrypt_digits(ref, sk))
    assert (dev.decode(digits).cpu() - vals).abs().max() < 1e-8


@gpu
def test_bfv_scale_round_on_cuda_matches_big_integers():
    cpu, dev = _bfv_pair()
    q, p = cpu.q, cpu.p
    gen = torch.Generator().manual_seed(9)
    x = torch.randint(0, q, (5, cpu.n), generator=gen, dtype=torch.int64)
    # residues whose p*x/q sits at a rounding half-way point or a multiple of q/p, and the ends of [0, q)
    d = q // p
    edges = [0, 1, q - 1, q // 2, q // 2 + 1, d, d + 1, (d + 1) // 2, (d - 1) // 2, (p // 2) * d, (p // 2 + 1) * d]
    x[0, : len(edges)] = torch.tensor(edges, dtype=torch.int64)
    got = ops.bfv_scale_round(x.cuda(), q, p).cpu()
    assert torch.equal(got, ops.bfv_scale_round(x, q, p))
    want = [((xi * p + q // 2) // q) % p for xi in x.reshape(-1).tolist()]
    want = [v - p if v > p // 2 else v for v in want]
    assert got.reshape(-1).tolist() == want


@gpu
@pytest.mark.parametrize("bit_count", [1, 16])
def test_bfv_multiply_on_cuda_matches_the_cpu_context(bit_count):
    """ct x ct with relinearisation: on CUDA the key switch is one fused kernel over one limb and
    ceil(54 / bit_count) digits (54 at bit_count 1)."""
    cpu, dev = _bfv_pair()
    sk, pk = cpu.keygen(seed=11)
    rlk = cpu.relin_keygen(sk, seed=12, bit_count=bit_count, size=5)
    assert rlk.keys.shape[0] == -(-cpu.q.bit_length() // bit_count)
    va = torch.tensor([1.5, -2.25, 7.0], dtype=torch.float64)
    vb = torch.tensor([-0.75, 3.0, 0.5], dtype=torch.float64)
    ca, cb = cpu.encrypt(va, pk, seed=1), cpu.encrypt(vb, pk, seed=2)
    ref = cpu.multiply(ca, cb, rlk)
    rlk_g = BFVRelinKey(rlk.keys.cuda(), rlk.bit_count, rlk.size)
    out, names = kernels_run(lambda: dev.multiply(ca.cuda(), cb.cuda(), rlk_g))
    assert ran(names, f"keyswitch2_kernel<{dev.logn}>"), sorted(names)
    assert_same_words(out, ref)
    assert torch.allclose(dev.decrypt(out, sk.cuda()).cpu(), va * vb, atol=1e-9)


# ---------------------------------------------------------------------------------------------- 7. concurrency
@gpu
def test_concurrent_encrypt2_at_n16384_equals_sequential(cta_budget):
    """Two N = 16384 encrypts on two streams, each under an encrypt budget of a third of the chip so that both are
    resident at once. Each keeps NTT(u) of its ciphertext in flight in a global scratch row per CTA; the rows must be
    private to the launch."""
    c, g = _ctx_pair(16384, (54, 54, 54, 54))
    _, pk = c.keygen(seed=81)
    pk_g = pk.cuda()
    budget = 2 * (_sms() // 6)
    gen = torch.Generator().manual_seed(82)
    with cta_budget(0, budget, 0):
        C = _count(4 * _max_workers(_grid(budget), c.L) + 1, c.logn)
        msgs = [torch.randint(-2**40, 2**40, (C, c.n), generator=gen, dtype=torch.int64) for _ in range(2)]
        refs = [ops.encrypt(m, pk, C, c.L, c.logn, c.tables, c.consts, None, 90 + i, i * C)
                for i, m in enumerate(msgs)]
        msgs_g = [m.cuda() for m in msgs]
        # sequential, under the profiler: the persistent kernel is the one that runs at this size and budget
        seq, names = kernels_run(lambda: [ops.encrypt(m, pk_g, C, c.L, c.logn, g.tables, g.consts, None, 90 + i, i * C)
                                          for i, m in enumerate(msgs_g)])
        assert ran(names, "encrypt2_kernel<14>"), sorted(names)
        for s, r in zip(seq, refs):
            assert_same_words(s, r)
        # concurrent: both streams wait on one spinning kernel, so the two launches are released together
        cur = torch.cuda.current_stream()
        streams = [torch.cuda.Stream() for _ in range(2)]
        torch.cuda.synchronize()
        torch.cuda._sleep(20_000_000)
        outs = []
        for i, (st, m) in enumerate(zip(streams, msgs_g)):
            st.wait_stream(cur)
            with torch.cuda.stream(st):
                outs.append(ops.encrypt(m, pk_g, C, c.L, c.logn, g.tables, g.consts, None, 90 + i, i * C))
        torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        assert_same_words(o, r)
