"""Property tests (hypothesis) over random ring degrees, limb counts and client counts, plus a
byte-level golden fixture of our own serialization format (SURVEY.md §4.3; Pyfhel 2.3.1 golden
ciphertexts cannot be produced offline — there is no Pyfhel/SEAL on this box)."""
import struct

import torch
from hypothesis import given, settings, strategies as st

from hefl_b200 import _ext
from hefl_b200.he.context import CKKSContext, CtBatch

ops = _ext.ops()
CFG = dict(max_examples=12, deadline=None)


@settings(**CFG)
@given(logn=st.integers(4, 9), L=st.integers(1, 3), seed=st.integers(0, 2**31 - 1))
def test_ntt_is_linear_and_invertible(logn, L, seed):
    n = 1 << logn
    primes = ops.gen_primes(45, logn, L, [])
    tables, consts = ops.build_tables(primes, logn)
    g = torch.Generator().manual_seed(seed)
    a = torch.stack([torch.randint(0, int(q), (n,), generator=g, dtype=torch.int64) for q in primes])
    b = torch.stack([torch.randint(0, int(q), (n,), generator=g, dtype=torch.int64) for q in primes])
    s = torch.empty_like(a)
    ops.pointwise_(s, a, b, L, consts, 0)
    fa, fb, fs = a.clone(), b.clone(), s.clone()
    for t in (fa, fb, fs):
        ops.ntt_(t, tables, consts, L, logn, False)
    chk = torch.empty_like(a)
    ops.pointwise_(chk, fa, fb, L, consts, 0)
    assert torch.equal(chk, fs)
    ops.ntt_(fs, tables, consts, L, logn, True)
    assert torch.equal(fs, s)


@settings(**CFG)
@given(logn=st.integers(5, 10), L=st.integers(1, 3), K=st.integers(1, 8), seed=st.integers(0, 2**31 - 1))
def test_additive_homomorphism_any_shape(logn, L, K, seed):
    n = 1 << logn
    ctx = CKKSContext(n, prime_bits=(45,) * L, scale_bits=30, enforce_security=False)
    sk, pk = ctx.keygen(seed=seed)
    g = torch.Generator().manual_seed(seed)
    nvals = n // 2 + 3
    ws = [torch.randn(nvals, generator=g) for _ in range(K)]
    acc = None
    for i, w in enumerate(ws):
        ct = ctx.encrypt(w, pk, seed=seed + i + 1)
        acc = ct if acc is None else ctx.add_(acc, ct)
    out = ctx.decrypt(acc, sk, divide_by=K)
    ref = torch.stack(ws).mean(0)
    assert (out - ref).abs().max() < 5e-3 * (1 + n / 256)


@settings(**CFG)
@given(K=st.integers(1, 12), L=st.integers(1, 4), seed=st.integers(0, 2**31 - 1))
def test_local_sum_matches_bigint(K, L, seed):
    logn, n = 4, 16
    primes = ops.gen_primes(60, logn, L, [])
    _, consts = ops.build_tables(primes, logn)
    g = torch.Generator().manual_seed(seed)
    srcs = [torch.stack([torch.randint(0, int(q), (2, n), generator=g, dtype=torch.int64) for q in primes], dim=1).contiguous()
            for _ in range(K)]
    out = torch.empty_like(srcs[0])
    ops.local_sum_modq(srcs, out, L, logn, consts)
    for l, q in enumerate(int(v) for v in primes):
        exp = [sum(int(s[c, l, i]) for s in srcs) % q for c in range(2) for i in range(n)]
        assert [int(v) for v in out[:, l].reshape(-1)] == exp


def test_local_sum_of_many_maximal_addends_under_61_bit_primes():
    """q - 1 from every source under primes just below 2^61: 8 of them sum to just below 2^64, so a reduced
    accumulator may take only 7 more before the next reduction."""
    logn, n, L = 10, 1024, 3
    primes = ops.gen_primes(61, logn, L, [])
    _, consts = ops.build_tables(primes, logn)
    top = torch.stack([torch.full((2, n), int(q) - 1, dtype=torch.int64) for q in primes], dim=1).contiguous()
    for K in (1, 7, 8, 9, 15, 16, 17, 24, 25, 64):
        out = torch.empty_like(top)
        ops.local_sum_modq([top] * K, out, L, logn, consts)
        for l, q in enumerate(int(v) for v in primes):
            assert torch.equal(out[:, l], torch.full((2, n), K * (q - 1) % q, dtype=torch.int64)), (K, l)


def test_serialization_golden_bytes():
    """Byte-level fixture of the HEFL stream header (format version 1)."""
    ctx = CKKSContext(4096, prime_bits=(36, 36, 37), scale_bits=40)
    blob = ctx.to_bytes_context()
    assert blob[:4] == b"HEFL"
    ver, kind, n, L, sb = struct.unpack_from("<HHIII", blob, 4)
    assert (ver, kind, n, L, sb) == (1, 1, 4096, 3, 40)
    assert list(struct.unpack_from("<3Q", blob, 20)) == [68719403009, 68719230977, 137438822401]
    assert blob.hex() == "4845464c0100010000100000030000002800000001e0feff0f0000000140fcff0f0000000100feff1f000000010000008000000000000000"
    ct = CtBatch(torch.arange(2 * 3 * 4096, dtype=torch.int64).view(1, 2, 3, 4096), ctx.scale, 7, "slots")
    raw = ctx.ct_to_bytes(ct)
    hdr = CKKSContext.parse_header(raw)
    assert hdr["kind"] == 4 and hdr["extra"][:5] == [4, 1, 2, 3, 4096] and hdr["extra"][6] == 7
    assert len(raw) == hdr["offset"] + 2 * 3 * 4096 * 8
    back = ctx.ct_from_bytes(raw)
    assert torch.equal(back.data, ct.data) and back.nvals == 7 and back.scale == ctx.scale


def test_reciprocal_division_used_by_the_conv_kernels_is_exact():
    """csrc/nn/conv_tcgen05.cu::fast_div replaces n / d by umulhi(n, ceil(2^32 / d)) for tile indices
    (n, d < 2^16, d > 1). The identity must hold for every value the host code allows."""
    import random
    rng = random.Random(0)
    ds = list(range(2, 600)) + [rng.randrange(2, 65536) for _ in range(300)] + [65535]
    for d in ds:
        magic = ((1 << 32) + d - 1) // d
        assert magic < (1 << 32)
        ns = [0, 1, d - 1, d, d + 1, 2 * d - 1, 65535, 65534] + [rng.randrange(0, 65536) for _ in range(64)]
        for n in ns:
            if n < 65536:                              # the host code only enables the magic for n < 2^16
                assert (n * magic) >> 32 == n // d, (n, d)
