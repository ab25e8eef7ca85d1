"""Packed-CKKS context, keys and ciphertext batches (the product HE surface).

What the reference does per scalar weight through Pyfhel/SEAL —
``HE.encryptFrac(weight[k])`` (FLPyfhelin.py:216-217), ``enc + dct`` (:381),
``dct * denom`` (:385), ``HE.decryptFrac`` (:295) — is done here on whole models at once:
a flat fp32 weight vector becomes a ``[C, 2, L, N]`` u64 tensor (C ciphertexts of N/2
slots, 2 polynomials, L RNS limbs, NTT form), so that FedAvg is one coefficient-wise
modular add-reduce (fused with the collective in ``hefl_b200.parallel``) and the 1/K factor
is folded into the decode scale (SURVEY.md §2.2 X1.h, §7.5).

All heavy lifting is in ``torch.ops.hefl`` (csrc/he): the same calls run the sm_90a
kernels for CUDA tensors and the host C++ implementation for CPU tensors.
"""
from __future__ import annotations

import dataclasses
import math
import struct
from typing import List, Optional, Sequence, Tuple

import torch

from .. import _ext
from ..config import SEC_MAX_LOGQ

MAGIC = b"HEFL"
FORMAT_VERSION = 1
KIND_CONTEXT, KIND_PUBLIC, KIND_SECRET, KIND_CIPHER, KIND_RELIN = 1, 2, 3, 4, 5


def _log2(n: int) -> int:
    l = n.bit_length() - 1
    if 1 << l != n:
        raise ValueError(f"ring degree must be a power of two, got {n}")
    return l


@dataclasses.dataclass
class CtBatch:
    """A batch of ciphertexts: ``data`` is int64 ``[C, 2, L, N]`` (u64 words, NTT form)."""

    data: torch.Tensor
    scale: float
    nvals: int
    packing: str = "slots"

    @property
    def count(self) -> int:
        return self.data.shape[0]

    @property
    def level(self) -> int:
        return self.data.shape[2]

    def clone(self) -> "CtBatch":
        return CtBatch(self.data.clone(), self.scale, self.nvals, self.packing)

    def nbytes(self) -> int:
        return self.data.numel() * 8


class CKKSContext:
    """RNS-CKKS parameters + device tables.

    Parameters mirror BASELINE.json configs: ``n=4096`` with three primes (36, 36, 37 bits),
    ``n=8192`` with four, ``n=16384``; primes are NTT-friendly (q = 1 mod 2N), < 2^61.
    """

    def __init__(self, n: int, prime_bits: Sequence[int] = (36, 36, 37), scale_bits: int = 40,
                 device: str | torch.device = "cpu", sec: int = 128, enforce_security: bool = True,
                 primes: Optional[Sequence[int]] = None):
        self.ops = _ext.ops()
        self.n = int(n)
        self.logn = _log2(self.n)
        if primes is None:
            primes = self._pick_primes(self.logn, list(prime_bits))
        self.primes: List[int] = [int(p) for p in primes]
        self.L = len(self.primes)
        self.scale = float(2.0 ** scale_bits)
        self.scale_bits = int(scale_bits)
        self.sec = int(sec)
        logq = sum(p.bit_length() for p in self.primes)
        if enforce_security and sec in SEC_MAX_LOGQ and self.n in SEC_MAX_LOGQ[sec]:
            if logq > SEC_MAX_LOGQ[sec][self.n]:
                raise ValueError(
                    f"log2(Q)={logq} exceeds the {sec}-bit security bound "
                    f"{SEC_MAX_LOGQ[sec][self.n]} for n={self.n}")
        self.logq = logq
        moduli = torch.tensor(self.primes, dtype=torch.int64)
        tables, consts = self.ops.build_tables(moduli, self.logn)
        rot, ksi = self.ops.build_fft_tables(self.logn)
        self._cpu = dict(tables=tables, consts=consts, rot=rot, ksi=ksi)
        self.consts_cpu = consts
        self.q0_inv_q1 = pow(self.primes[0], -1, self.primes[1]) if self.L > 1 else 0
        self.device = torch.device("cpu")
        self._limb_cache = {}
        self.tables, self.consts, self.rot, self.ksi = tables, consts, rot, ksi
        self.to(device)

    # ------------------------------------------------------------------ parameters
    def _pick_primes(self, logn: int, bits: List[int]) -> List[int]:
        chosen: List[int] = []
        for b in bits:
            p = self.ops.gen_primes(b, logn, 1, chosen)
            chosen.append(int(p[0]))
        return chosen

    def to(self, device: str | torch.device) -> "CKKSContext":
        device = torch.device(device)
        self.device = device
        self.tables = self._cpu["tables"].to(device)
        self.consts = self._cpu["consts"].to(device)
        self.rot = self._cpu["rot"].to(device)
        self.ksi = self._cpu["ksi"].to(device)
        return self

    @property
    def slots(self) -> int:
        return self.n // 2

    def values_per_ct(self, packing: str = "slots") -> int:
        return self.n // 2 if packing == "slots" else self.n

    def num_ct(self, nvals: int, packing: str = "slots") -> int:
        v = self.values_per_ct(packing)
        return (nvals + v - 1) // v

    def ct_bytes(self, level: Optional[int] = None) -> int:
        return 2 * (level or self.L) * self.n * 8

    def max_abs_message(self, k_limbs: Optional[int] = None) -> float:
        """Largest |value * scale * K| the 1- or 2-limb device decode can represent."""
        k = min(self.L, 2) if k_limbs is None else k_limbs
        q = 1
        for p in self.primes[:k]:
            q *= p
        return q / 4.0

    # ------------------------------------------------------------------ keys
    def _key_tables(self):
        """(tables, consts) for key generation: the device copies on CUDA (kernels in he_kernels.cu), the host twin
        otherwise. Both produce the same keys for a given seed."""
        if self.device.type == "cuda":
            return self.tables, self.consts
        return self._cpu["tables"], self._cpu["consts"]

    def keygen(self, seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """Returns (sk [L,N], pk [2,L,N]) on the context device, generated there (HE.keyGen(), FLPyfhelin.py:340)."""
        t, c = self._key_tables()
        sk = self.ops.keygen_secret(self.L, self.logn, t, c, int(seed))
        pk = self.ops.keygen_public(sk, self.L, self.logn, t, c, int(seed), 0)
        return sk.to(self.device), pk.to(self.device)

    def relin_keygen(self, sk: torch.Tensor, seed: int = 0, digit_bits: int = 16) -> "RelinKey":
        """Digit-decomposed evaluation key for s^2 -> s (SURVEY.md K10; FLPyfhelin.py:357-364).

        evk[i][k] = (-(a s + e) + 2^(k*digit_bits) * g_i * s^2, a) where g_i is the CRT basis
        element of limb i (1 mod q_i, 0 mod q_j): limb j of the message term is non-zero only
        for j == i. All digits of all limbs are generated by one batched call (sample, NTT, finish) and one
        message-term kernel, on the context device.
        """
        t, c = self._key_tables()
        sk_d = sk.to(t.device).contiguous()
        s2 = torch.empty_like(sk_d)
        self.ops.pointwise_(s2, sk_d, sk_d, self.L, c, 2)
        nd = [(self.primes[i].bit_length() + digit_bits - 1) // digit_bits for i in range(self.L)]
        limb_of = [i for i in range(self.L) for _ in range(nd[i])]
        w = [pow(2, k * digit_bits, self.primes[i]) for i in range(self.L) for k in range(nd[i])]
        evk = self.ops.keygen_public_batch(sk_d, self.L, self.logn, t, c, int(seed), 1, len(w))
        self.ops.relin_message_(evk, s2, torch.tensor(limb_of, dtype=torch.int32, device=t.device),
                                torch.tensor(w, dtype=torch.int64, device=t.device), self.L, c)
        evk = evk.to(self.device)
        keys, first = [], 0
        for i in range(self.L):
            keys.append(evk[first: first + nd[i]])
            first += nd[i]
        rlk = RelinKey(keys, digit_bits)
        rlk._flat = (evk, nd, [sum(nd[:i]) for i in range(self.L)])
        return rlk

    @staticmethod
    def _flat_evk(rlk: "RelinKey"):
        """[E, 2, L, N] evaluation keys + per-source-limb (digit count, first entry) for the fused key switch."""
        if getattr(rlk, "_flat", None) is None:
            nd = [int(k.shape[0]) for k in rlk.keys]
            first, acc = [], 0
            for d in nd:
                first.append(acc)
                acc += d
            rlk._flat = (torch.cat(list(rlk.keys), dim=0).contiguous(), nd, first)
        return rlk._flat

    # ------------------------------------------------------------------ encode / encrypt
    def encode(self, vals: torch.Tensor, packing: str = "slots", scale: Optional[float] = None,
               count: Optional[int] = None) -> torch.Tensor:
        """Flat real vector -> message polynomials int64 [C, N] (signed, coefficient form)."""
        vals = vals.reshape(-1).contiguous()
        if vals.dtype not in (torch.float32, torch.float64):
            vals = vals.float()
        C = count if count is not None else self.num_ct(vals.numel(), packing)
        sc = self.scale if scale is None else scale
        if packing == "slots":
            return self.ops.ckks_encode(vals, C, self.logn, sc, self.rot, self.ksi)
        if packing == "coeff":
            return self.ops.coeff_encode(vals.float(), C, self.n, sc)
        raise ValueError(f"unknown packing {packing}")

    def encrypt(self, vals: torch.Tensor, pk: torch.Tensor, seed: int, packing: str = "slots",
                out: Optional[torch.Tensor] = None, ct_offset: int = 0, weight: float = 1.0,
                accumulate: bool = False) -> CtBatch:
        """encode + public-key encrypt; ``out`` may be a view of a symmetric-memory buffer. ``weight`` multiplies
        the values inside the encode (scale Δ·weight) at no cost: the ciphertext carries weight·vals at scale Δ
        (sample-weighted FedAvg). ``weight=1.0`` encodes exactly as without it. ``accumulate=True`` adds the new
        ciphertexts into ``out`` mod q (out = out + Enc(vals)) in the encryption's own store, so the clients of one
        rank sum their updates without a buffer per client."""
        if accumulate and out is None:
            raise ValueError("accumulate=True adds into an existing ciphertext buffer: pass it as out=")
        nvals = vals.numel()
        msg = self.encode(vals, packing, scale=self.scale * float(weight))
        C = msg.shape[0]
        if out is None:
            data = self.ops.encrypt(msg, pk, C, self.L, self.logn, self.tables, self.consts, None,
                                    int(seed), int(ct_offset))
        else:
            data = out
            self.ops.encrypt_out(msg, pk, C, self.L, self.logn, self.tables, self.consts, None,
                                 int(seed), int(ct_offset), data, bool(accumulate))
            data = data.view(-1)[: C * 2 * self.L * self.n].view(C, 2, self.L, self.n)
        return CtBatch(data, self.scale, nvals, packing)

    def encrypt_zero(self, count: int, pk: torch.Tensor, seed: int) -> CtBatch:
        data = self.ops.encrypt(None, pk, count, self.L, self.logn, self.tables, self.consts, None,
                                int(seed), 0)
        return CtBatch(data, self.scale, 0, "slots")

    # ------------------------------------------------------------------ decrypt / decode
    def decrypt_residues(self, ct: CtBatch, sk: torch.Tensor, k: Optional[int] = None) -> torch.Tensor:
        k = min(ct.level, 2) if k is None else k
        return self.ops.decrypt(ct.data, sk, k, self.logn, self.tables, self.consts)

    def decrypt(self, ct: CtBatch, sk: torch.Tensor, divide_by: float = 1.0) -> torch.Tensor:
        """Ciphertext batch -> flat fp32 vector of ``ct.nvals`` values, divided by ``divide_by``
        (the FedAvg 1/K, folded into the decode scale at zero cost)."""
        res = self.decrypt_residues(ct, sk)
        inv = 1.0 / (ct.scale * divide_by)
        if ct.packing == "slots":
            return self.ops.ckks_decode_residues(res, self.consts_cpu, self.q0_inv_q1, self.logn,
                                                 inv, self.rot, self.ksi, ct.nvals)
        coeffs = self.ops.crt_center(res, self.consts_cpu, self.q0_inv_q1)
        return (coeffs.reshape(-1)[: ct.nvals] * inv).float()

    def decrypt_server_step(self, ct: CtBatch, sk: torch.Tensor, divide_by: float, x_t: torch.Tensor,
                            x_new: torch.Tensor, m: torch.Tensor, v: torch.Tensor, opt, hp, n_trainable: int,
                            offset: int = 0, avg_out: Optional[torch.Tensor] = None) -> None:
        """``decrypt`` fused with a server-optimizer step (hefl_b200.fl.server_opt, DESIGN.md §8): the batch holds
        flat values ``offset .. offset + ct.nvals - 1`` of a model; for each, the decoded average ``a`` and the
        round's starting weight ``x_t[g]`` give ``x_new[g]``, and ``m`` / ``v`` (``n_trainable`` fp32 entries) are
        updated in place. ``opt`` is a name or code of ``SERVER_OPTS`` (not fedavg); ``hp`` holds lr, beta1,
        beta2 and tau. ``avg_out`` (fp32 or fp64, indexed like ``x_new``) also receives the average."""
        if ct.packing != "slots":
            raise ValueError("the server-optimizer step is fused into the slot decode; coefficient packing is "
                             "not supported")
        if isinstance(opt, str):
            from ..fl.server_opt import SERVER_OPTS
            opt = SERVER_OPTS[opt]
        res = self.decrypt_residues(ct, sk)
        inv = 1.0 / (ct.scale * divide_by)
        self.ops.ckks_decode_server_step_(res, self.consts_cpu, self.q0_inv_q1, self.logn, inv, self.rot, self.ksi,
                                          ct.nvals, int(offset), int(n_trainable), x_t, x_new, m, v, int(opt),
                                          float(hp["lr"]), float(hp["beta1"]), float(hp["beta2"]), float(hp["tau"]),
                                          avg_out)

    def decode(self, coeffs: torch.Tensor, scale: float, as_f64: bool = False) -> torch.Tensor:
        return self.ops.ckks_decode(coeffs.contiguous(), self.logn, 1.0 / scale, self.rot, self.ksi, as_f64)

    # ------------------------------------------------------------------ homomorphic ops
    def add_(self, a: CtBatch, b: CtBatch) -> CtBatch:
        self._check_compatible(a, b)
        self.ops.pointwise_(a.data, a.data, b.data, a.level, self.consts, 0)
        return a

    def add(self, a: CtBatch, b: CtBatch) -> CtBatch:
        return self.add_(a.clone(), b)

    def sub_(self, a: CtBatch, b: CtBatch) -> CtBatch:
        self._check_compatible(a, b)
        self.ops.pointwise_(a.data, a.data, b.data, a.level, self.consts, 1)
        return a

    def negate_(self, a: CtBatch) -> CtBatch:
        self.ops.pointwise_(a.data, a.data, None, a.level, self.consts, 4)
        return a

    def sum_batches(self, batches: Sequence[CtBatch]) -> CtBatch:
        """Server-side aggregation without keys (FLPyfhelin.py:372-381)."""
        acc = batches[0].clone()
        for b in batches[1:]:
            self.add_(acc, b)
        return acc

    def add_plain_(self, a: CtBatch, vals: torch.Tensor) -> CtBatch:
        """ct + plaintext vector (X1.g): encode at the ciphertext scale, NTT, add into c0."""
        msg = self.encode(vals.to(self.device), a.packing, scale=a.scale, count=a.count)
        pt = self._msg_to_ntt(msg, a.level)
        c0 = a.data[:, 0]
        tmp = c0.contiguous()
        self.ops.pointwise_(tmp, tmp, pt, a.level, self.consts, 0)
        a.data[:, 0] = tmp
        return a

    def mul_scalar_(self, a: CtBatch, value: float, rescale: bool = True) -> CtBatch:
        """ct * real constant (FLPyfhelin.py:385 ``* denom``): the constant is encoded at scale
        q_last so that the following rescale returns exactly to the input scale."""
        lvl = a.level
        if rescale and lvl < 2:
            raise ValueError("cannot rescale a level-1 ciphertext")
        q_last = self.primes[lvl - 1]
        csc = float(q_last) if rescale else self.scale
        c_int = int(round(value * csc))
        scal = torch.tensor([c_int % self.primes[l] for l in range(lvl)], dtype=torch.int64,
                            device=self.device)
        self.ops.pointwise_(a.data, a.data, scal, lvl, self.consts, 5)
        a.scale = a.scale * csc
        if rescale:
            self.rescale_(a)
        return a

    def mul_plain_(self, a: CtBatch, vals: torch.Tensor, rescale: bool = True) -> CtBatch:
        """Slot-wise ct * plaintext vector (K9)."""
        lvl = a.level
        q_last = self.primes[lvl - 1]
        psc = float(q_last) if rescale else self.scale
        msg = self.encode(vals.to(self.device), a.packing, scale=psc, count=a.count)
        pt = self._msg_to_ntt(msg, lvl)  # [C, L, N]
        for j in range(2):
            cj = a.data[:, j].contiguous()
            self.ops.pointwise_(cj, cj, pt, lvl, self.consts, 2)
            a.data[:, j] = cj
        a.scale *= psc
        if rescale:
            self.rescale_(a)
        return a

    def rescale_(self, a: CtBatch) -> CtBatch:
        """Drop the last limb with rounding: ct <- round(ct / q_last) (K9)."""
        lvl = a.level
        if lvl < 2:
            raise ValueError("no limb left to drop")
        C = a.count
        ql = self.primes[lvl - 1]
        if a.data.is_cuda:
            # one fused launch (csrc/he/cuda/he_eval2.cu): INTT of the last limb -> centred lift -> NTT under every
            # remaining prime -> subtract -> * q_last^-1
            out = self.ops.rescale_fused(a.data.contiguous(), self.tables, self.consts, self.consts_cpu, self.logn)
            if out.numel() or C == 0:
                a.data = out if out.numel() else a.data[:, :, :lvl - 1].contiguous()
                a.scale = a.scale / float(ql)
                return a
        # reference path (CPU tensors, N >= 16384, primes >= 2^58): the same steps, limb by limb
        # last limb to coefficient form
        last = a.data[:, :, lvl - 1].contiguous()            # [C,2,N]
        self._ntt_single_limb(last, lvl - 1, inverse=True)
        half = ql // 2
        last = torch.remainder(last + half, ql)              # [c_last + q_last/2]_{q_last}
        out = torch.empty(C, 2, lvl - 1, self.n, dtype=torch.int64, device=self.device)
        for j in range(lvl - 1):
            qj = self.primes[j]
            # t = ([c + half]_{q_last} - half) mod q_j, then NTT under q_j  (centred rounding)
            t = torch.remainder(torch.remainder(last, qj) - (half % qj), qj).contiguous()
            self._ntt_single_limb(t, j, inverse=False)
            cj = a.data[:, :, j].contiguous()
            diff = torch.empty_like(cj)
            self._pointwise_limb(diff, cj, t, j, 1)
            inv = pow(ql, -1, qj)
            self._scalar_limb(diff, diff, inv, j)
            out[:, :, j] = diff
        a.data = out
        a.scale = a.scale / float(ql)
        return a

    def multiply(self, a: CtBatch, b: CtBatch, rlk: "RelinKey", rescale: bool = True) -> CtBatch:
        """ct * ct with relinearisation (API parity: PyCtxt * PyCtxt, SURVEY.md K10)."""
        self._check_compatible(a, b, same_scale=False)
        lvl = a.level
        if a.data.is_cuda and lvl == self.L and rlk is not None:
            # fused path: one tensor-product kernel, one batched INTT, one key-switch kernel that accumulates
            # every (source limb, digit) term in shared memory on top of (d0, d1)
            d01, d2 = self.ops.ct_tensor(a.data.contiguous(), b.data.contiguous(), self.consts)
            self.ops.ntt_(d2, self.tables, self.consts, lvl, self.logn, True)
            evk, nd, first = self._flat_evk(rlk)
            if self.ops.keyswitch_fused_(d01, d2, evk, nd, first, rlk.digit_bits, self.tables, self.consts, self.logn):
                out = CtBatch(d01, a.scale * b.scale, min(a.nvals, b.nvals), a.packing)
                if rescale:
                    self.rescale_(out)
                return out
        a0, a1 = a.data[:, 0].contiguous(), a.data[:, 1].contiguous()
        b0, b1 = b.data[:, 0].contiguous(), b.data[:, 1].contiguous()
        d0 = torch.empty_like(a0)
        d1 = torch.empty_like(a0)
        d2 = torch.empty_like(a0)
        self.ops.pointwise_(d0, a0, b0, lvl, self.consts, 2)
        self.ops.pointwise_(d1, a0, b1, lvl, self.consts, 2)
        self.ops.pointwise_(d1, a1, b0, lvl, self.consts, 3)
        self.ops.pointwise_(d2, a1, b1, lvl, self.consts, 2)
        r0, r1 = self._keyswitch(d2, rlk, lvl)
        self.ops.pointwise_(d0, d0, r0, lvl, self.consts, 0)
        self.ops.pointwise_(d1, d1, r1, lvl, self.consts, 0)
        out = CtBatch(torch.stack([d0, d1], dim=1).contiguous(), a.scale * b.scale,
                      min(a.nvals, b.nvals), a.packing)
        if rescale:
            self.rescale_(out)
        return out

    # ------------------------------------------------------------------ internals
    def _keyswitch(self, d2: torch.Tensor, rlk: "RelinKey", lvl: int):
        """sum_{i,k} digit_{i,k}(d2) * evk[i][k]; d2 is [C, L, N] in NTT form."""
        C = d2.shape[0]
        coef = d2.clone()
        self.ops.ntt_(coef, self.tables, self.consts, lvl, self.logn, True)
        r0 = torch.zeros_like(d2)
        r1 = torch.zeros_like(d2)
        for i in range(lvl):
            src = coef[:, i].contiguous()                     # [C, N] residues mod q_i
            for k in range(rlk.keys[i].shape[0]):
                dig = self.ops.digit_extract(src, k * rlk.digit_bits, rlk.digit_bits)  # [C,N]
                ext = dig.unsqueeze(1).expand(C, lvl, self.n).contiguous()
                self.ops.ntt_(ext, self.tables, self.consts, lvl, self.logn, False)
                ek = rlk.keys[i][k]                           # [2, L, N]
                self.ops.pointwise_(r0, ext, ek[0, :lvl].contiguous(), lvl, self.consts, 3)
                self.ops.pointwise_(r1, ext, ek[1, :lvl].contiguous(), lvl, self.consts, 3)
        return r0, r1

    def _limb_views(self, limb: int):
        # cached: the native layer keys its derived (interleaved) tables on these tensors
        key = (limb, str(self.device))
        v = self._limb_cache.get(key)
        if v is None:
            v = (self.tables[limb:limb + 1].contiguous(), self.consts[limb:limb + 1].contiguous())
            self._limb_cache[key] = v
        return v

    def _ntt_single_limb(self, x: torch.Tensor, limb: int, inverse: bool) -> None:
        t, c = self._limb_views(limb)
        self.ops.ntt_(x, t, c, 1, self.logn, inverse)

    def _pointwise_limb(self, out, a, b, limb: int, op: int) -> None:
        _, c = self._limb_views(limb)
        self.ops.pointwise_(out, a, b, 1, c, op)

    def _scalar_limb(self, out, a, value: int, limb: int) -> None:
        _, c = self._limb_views(limb)
        s = torch.tensor([value], dtype=torch.int64, device=self.device)
        self.ops.pointwise_(out, a, s, 1, c, 5)

    def _msg_to_ntt(self, msg: torch.Tensor, lvl: int) -> torch.Tensor:
        """Signed message [C,N] -> residues [C,lvl,N] in NTT form."""
        C = msg.shape[0]
        limbs = []
        for l in range(lvl):
            limbs.append(torch.remainder(msg, self.primes[l]))
        pt = torch.stack(limbs, dim=1).contiguous()
        self.ops.ntt_(pt, self.tables, self.consts, lvl, self.logn, False)
        return pt

    def _check_compatible(self, a: CtBatch, b: CtBatch, same_scale: bool = True) -> None:
        if a.data.shape != b.data.shape:
            raise ValueError(f"ciphertext shapes differ: {tuple(a.data.shape)} vs {tuple(b.data.shape)}")
        if same_scale and not math.isclose(a.scale, b.scale, rel_tol=1e-9):
            raise ValueError("ciphertext scales differ")

    # ------------------------------------------------------------------ serialization (K12)
    def _header(self, kind: int, extra: Sequence[int] = ()) -> bytes:
        h = MAGIC + struct.pack("<HHIII", FORMAT_VERSION, kind, self.n, self.L, self.scale_bits)
        h += struct.pack(f"<{self.L}Q", *self.primes)
        h += struct.pack("<I", len(extra)) + struct.pack(f"<{len(extra)}q", *extra)
        return h

    def to_bytes_context(self) -> bytes:
        return self._header(KIND_CONTEXT, (self.sec,))

    @staticmethod
    def parse_header(buf: bytes):
        if buf[:4] != MAGIC:
            raise ValueError("not a hefl_b200 stream")
        ver, kind, n, L, sb = struct.unpack_from("<HHIII", buf, 4)
        if ver != FORMAT_VERSION:
            raise ValueError(f"unsupported stream version {ver}")
        off = 4 + 16
        primes = list(struct.unpack_from(f"<{L}Q", buf, off))
        off += 8 * L
        (ne,) = struct.unpack_from("<I", buf, off)
        off += 4
        extra = list(struct.unpack_from(f"<{ne}q", buf, off))
        off += 8 * ne
        return dict(kind=kind, n=n, L=L, scale_bits=sb, primes=primes, extra=extra, offset=off)

    @classmethod
    def from_bytes_context(cls, buf: bytes, device: str | torch.device = "cpu") -> "CKKSContext":
        h = cls.parse_header(buf)
        if h["kind"] != KIND_CONTEXT:
            raise ValueError("stream is not a context")
        return cls(h["n"], primes=h["primes"], scale_bits=h["scale_bits"], device=device,
                   sec=h["extra"][0] if h["extra"] else 128, enforce_security=False)

    def tensor_to_bytes(self, t: torch.Tensor, kind: int, extra: Sequence[int] = ()) -> bytes:
        shape = list(t.shape)
        body = t.detach().cpu().contiguous().numpy().tobytes()
        return self._header(kind, [len(shape), *shape, *extra]) + body

    def tensor_from_bytes(self, buf: bytes, kind: int):
        h = self.parse_header(buf)
        if h["kind"] != kind:
            raise ValueError(f"stream kind {h['kind']} != expected {kind}")
        if h["n"] != self.n or h["primes"] != self.primes:
            raise ValueError("stream was produced under different HE parameters")
        nd = h["extra"][0]
        shape = h["extra"][1:1 + nd]
        rest = h["extra"][1 + nd:]
        import numpy as np

        arr = np.frombuffer(buf, dtype=np.int64, offset=h["offset"]).reshape(shape).copy()
        return torch.from_numpy(arr).to(self.device), rest

    def ct_to_bytes(self, ct: CtBatch) -> bytes:
        sc = struct.unpack("<q", struct.pack("<d", ct.scale))[0]
        return self.tensor_to_bytes(ct.data, KIND_CIPHER, [sc, ct.nvals, 0 if ct.packing == "slots" else 1])

    def ct_from_bytes(self, buf: bytes) -> CtBatch:
        data, rest = self.tensor_from_bytes(buf, KIND_CIPHER)
        scale = struct.unpack("<d", struct.pack("<q", rest[0]))[0]
        return CtBatch(data, scale, int(rest[1]), "slots" if rest[2] == 0 else "coeff")

    def __repr__(self) -> str:
        bits = "+".join(str(p.bit_length()) for p in self.primes)
        return (f"<CKKSContext n={self.n} L={self.L} logQ={self.logq} ({bits}) "
                f"scale=2^{self.scale_bits} sec={self.sec} device={self.device}>")


@dataclasses.dataclass
class RelinKey:
    keys: List[torch.Tensor]   # per limb i: [digits_i, 2, L, N]
    digit_bits: int
