"""Both attention kernels against an fp64 reference, at every head dim, ragged edge, shared slot and weight table.

The attention core (softmax(q k^T / sqrt(hd)) with optional post-softmax weights on the last keys, times v) has two kernels:
the wgmma + TMA kernel (csrc/attention_wg.cu) runs head_dim 80, the mma.sync kernel (csrc/attention.cu) every other head
dim, and head_dim 80 too with PB200_ATTN_MMA_SYNC=1.  That knob is read once per process, so the mma.sync kernel's head_dim-80
cases run in a child process; everything else runs in-process.  Every case goes through pb200_attention_slots, which reaches
every AttnParams field (kv_len, kv_slot, n_slots and the per-sample weight table), and checks:
  * element by element against fp64 arithmetic on the same fp16 inputs:
        |got - ref| <= U16 |ref| + TAU_P sum_j p_j |v_j| + TAU_S L_i (sum_j p_j |v_j| + |ref|) + Nk 2^-25 max_j |v_j|
    with p_j the fp64 weight of key j (after attn_weights), U16 = 2^-11 the fp16 store, TAU_P the fp16 rounding of P and the
    fp32 accumulation, L_i = log2(e) max_j (|z_j| + |z_max| + sum_d |q_d k_jd| / sqrt(hd)) the size of the fp32 exponent
    arithmetic of row i (z = q k / sqrt(hd)), and the last term fp16-subnormal P;
  * that the bound can see a wrong kernel: probe keys k_j = alpha q_i planted on the last valid key, the first masked key,
    chunk and 16-key group boundaries and the first and last weighted keys make dropping the last valid key, reading the first
    masked one, dropping the last 16-key group, shifting the weight window by one key and renormalising after the weights each
    move some element by at least SENS_MIN times its bound (computed in fp64);
  * isolation: rows a sample must not read (conditioning rows past kv_len, unreferenced slots, weight-table padding, and in
    dedicated cases every other sample's qkv) hold NaN, then +-Inf, and the output stays bit-identical; each checked sample
    also gives bit-identical output when run alone at B = 1 with its own copy of its slot;
  * the output sits inside a guard-banded buffer prefilled with a sentinel: every logical element is written, nothing outside
    changes, and a second launch is bit-identical;
  * shared slots give the output of each sample owning a copy of its slot, an all-equal weight table gives the single
    vector's output, and a row of length 0 (or a sample past w_batch) gives the unweighted output, all bit for bit.
Refusals (unsupported head dims, E % nhead != 0) return an error and leave the output untouched; B = 0 and P = 0 do nothing.
One row per case (kernel, case, error/bound, sensitivity) is appended to attention_matrix.jsonl in $PB200_TEST_LOG_DIR (see
helpers.log_jsonl).
"""
import ctypes
import json
import math
import os
import subprocess
import sys
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# Calibrated on an H100 80GB HBM3 (700 W power limit).  Each term alone (the other set to 0) would have to be: TAU_P 2^-11.4
# on every case (the fp16 rounding of P, at most 2^-11), TAU_S 2^-21.1 on the large-logit cases, where L_i reaches ~700 and
# the exponent term dominates the bound.  TAU_P = 2^-10 and TAU_S = 2^-20 keep 2.7x and 2.1x margins over those.  The worst
# error/bound per kernel at these values is WORST_OBSERVED: above 0.5 because the fp16 store's half-ulp is in both the error
# and the bound (0.32 at most on the large-logit cases).  The smallest sensitivity was 188 (renormalising a 1-entry weight
# vector at large logits).
TAU_P = 2.0 ** -10
TAU_S = 2.0 ** -20
WORST_OBSERVED = {"wgmma": 0.522, "mma.sync hd80": 0.522, "mma.sync": 0.550}
SENS_MIN = 20.0
U16 = 2.0 ** -11
LOG2E = 1.4426950408889634
SENTINEL = 0x7E5A                        # an fp16 NaN pattern no finite output has
KERNELS = ("wgmma", "mma80", "mma")      # mma80: head_dim 80 through the mma.sync kernel (child process)
BIG_ELEMS = 2 ** 31


def _log(payload):
    from helpers import log_jsonl
    log_jsonl("attention_matrix.jsonl", payload)


# ------------------------------------------------------------------ the case matrix
def _cases(kernel):
    """Each edge once per kernel, not as a full cross product.  hd None = 80 on the head_dim-80 kernels, and on the mma.sync
    kernel one of 16 / 32 / 64 / 96 in turn."""
    cases = []

    def add(name, B, P, H, S, self_=True, hd=None, **kw):
        cases.append(dict(name=name, B=B, P=P, H=H, S=S, self=self_, hd=hd, **kw))

    # ---- key counts: self only, conditioning only, both; 1, 63, 64, 65, 128, 129 and ~1100 keys
    add("self-P1", 3, 1, 2, 0)
    add("self-P63", 5, 63, 1, 0)
    add("self-P64", 2, 64, 16, 0)
    add("self-P65-vec5", 3, 65, 2, 0, weights=("vec", 5))
    add("self-P256-big-logits", 2, 256, 2, 0, logits="big")
    add("cond-P15-S1", 4, 15, 2, 1, self_=False)
    add("cond-P17-S63", 3, 17, 1, 63, self_=False, kv_len="full")
    add("cond-P64-S129-varlen", 4, 64, 2, 129, self_=False, kv_len=[128, 129, 64, 65])
    add("cond-P100-S1100-18chunks", 2, 100, 2, 1100, self_=False, kv_len=[1100, 1037], logits="big")
    add("both-P64-S64", 4, 64, 16, 64)
    add("both-P64-S65", 3, 64, 2, 65, logits="big")
    add("both-P100-S37-midchunk-vecncond", 3, 100, 2, 37, weights=("vec", 37))
    add("both-P256-S844-1100keys", 2, 256, 2, 844, kv_len=[844, 779])
    # ---- kv_len: 0 with self keys, 1, 63, 64, 65, s_max, varying across a batch of 300
    add("both-P16-S48-B300-varlen", 300, 16, 2, 48, kv_len="random0")
    add("both-P1-S64-B37-varlen", 37, 1, 1, 64, kv_len=[1, 63, 64])
    add("both-P65-S70-kvlen-edges", 5, 65, 2, 70, kv_len=[63, 64, 65, 70, 1])
    # ---- shared slots: several samples on one slot, a non-identity order, n_slots below and above B, the last slot read
    add("slots-below-B", 6, 65, 2, 70, slots=(3, [2, 0, 2, 1, 0, 2]), kv_len=[63, 70, 65])
    add("slots-above-B", 3, 17, 2, 40, slots=(7, [6, 3, 3]), kv_len=[5, 9, 13, 40, 2, 1, 33])
    add("slots-cond-only-last", 4, 64, 16, 132, self_=False, slots=(2, [1, 1, 0, 1]), kv_len=[132, 70])
    # ---- weights: one vector (n_w 1, 5, n_cond, past n_cond into the self keys, Nk), w_batch < B, tables
    add("vec-nw1-big-logits", 4, 64, 16, 132, weights=("vec", 1), logits="big")
    add("vec-nw-past-ncond", 3, 63, 2, 10, weights=("vec", 30))
    add("vec-nw-Nk-wbatch2", 4, 15, 2, 20, weights=("vec", 35, 2))
    add("table-w_row-shared", 8, 16, 2, 77, kv_len=[77, 50, 77, 20, 3, 70, 1, 40], weights=("table", [0, 5, 60, 93, 17], [3, 0, 3, 1, 4, 2], 100))
    add("table-slots", 5, 64, 16, 132, slots=(2, [1, 1, 0, 1, 0]), kv_len=[132, 100],
        weights=("table", [40, 0, 196, 7, 1], None, 200))
    # ---- every other sample's qkv poisoned
    add("isolate-qkv-P16", 4, 16, 2, 40, kv_len=[40, 3, 17, 40], isolate_qkv=True)
    add("isolate-qkv-self-P17", 5, 17, 1, 0, isolate_qkv=True)
    # ---- the shapes of the previous attention test (BASELINE configs 2 and 4 and their ragged / many-sample variants)
    add("cfg2-level1", 4, 64, 16, 132, hd=80)
    add("cfg2-level2-varlen", 3, 16, 16, 132, hd=80, kv_len="half")
    add("cfg4-level1-varlen", 2, 256, 16, 136, hd=80, kv_len="half")
    add("cfg4-level2-vec5", 2, 64, 16, 136, hd=80, weights=("vec", 5))
    add("cross-only-ragged", 5, 64, 4, 20, self_=False, hd=80, kv_len="half")
    add("two-query-tiles-S7", 2, 128, 2, 7, hd=80)
    add("cfg2-B160", 160, 64, 16, 132, hd=80)
    add("ragged-S100", 6, 64, 4, 100, hd=80, kv_len="half")
    add("P32-S12", 3, 32, 2, 12, hd=80)
    add("S190-254keys", 2, 64, 16, 190, hd=80, kv_len="half")
    add("cfg2-B300-varlen", 300, 64, 16, 132, hd=80, kv_len="half")
    add("hd16-P64-S9", 2, 64, 4, 9, hd=16)
    add("hd32-P16-S20-varlen-vec5", 2, 16, 4, 20, hd=32, kv_len="half", weights=("vec", 5))
    add("hd64-P100-S30", 2, 100, 2, 30, hd=64)
    other = (16, 32, 64, 96)
    out = []
    for i, c in enumerate(cases):
        if kernel == "mma":
            if c["hd"] == 80:
                continue
            c = dict(c, hd=c["hd"] or other[i % 4])
        else:
            if c["hd"] not in (None, 80):
                continue
            c = dict(c, hd=80)
        c["id"] = f"{c['name']}-hd{c['hd']}"
        out.append(c)
    ids = [c["id"] for c in out]
    assert len(ids) == len(set(ids))
    return out


# ------------------------------------------------------------------ inputs
def _kv_len_values(c, n_slots, gen):
    spec, S = c.get("kv_len"), c["S"]
    if spec is None or S == 0:
        return None
    if spec == "full":
        return [S] * n_slots
    if isinstance(spec, list):                   # repeated over the slots
        return [spec[i % len(spec)] for i in range(n_slots)]
    lo = {"half": max(1, S // 2), "random0": 0, "random1": 1}[spec]
    v = torch.randint(lo, S + 1, (n_slots,), generator=gen).tolist()
    v[0] = S
    if spec == "random0":
        v[1:4] = [0, 1, S - 1]
    return v


def _make(c):
    """Inputs, the per-sample key lists and the probes of case c (every tensor on the GPU, fp16 where the kernel reads fp16)."""
    B, P, H, S, hd = c["B"], c["P"], c["H"], c["S"], c["hd"]
    E = H * hd
    seed = zlib.crc32(c["id"].encode())
    gen = torch.Generator().manual_seed(seed)
    ggen = torch.Generator(device=DEV).manual_seed(seed)
    n_self = P if c["self"] else 0
    n_slots, kv_slot = (c["slots"][0], list(c["slots"][1])) if c.get("slots") else (B if S else 0, None)
    slot_of = kv_slot if kv_slot is not None else list(range(B))
    kv_len = _kv_len_values(c, n_slots, gen)
    n_cond = [(kv_len[s] if kv_len is not None else S) for s in slot_of] if S else [0] * B
    Nk = [n_self + n for n in n_cond]
    qscale = 15.0 if c.get("logits") == "big" else 1.0
    qkv = torch.randn(B * P, 3 * E, device=DEV, generator=ggen) * 1.5
    qkv[:, :E] *= qscale
    qkv = qkv.half()
    ckv = (torch.randn(n_slots, S, 2 * E, device=DEV, generator=ggen) * 1.5).half() if S else None
    s = dict(c=c, B=B, P=P, H=H, S=S, hd=hd, E=E, n_self=n_self, n_slots=n_slots, kv_slot=kv_slot, slot_of=slot_of,
             kv_len=kv_len, n_cond=n_cond, Nk=Nk, qkv=qkv, ckv=ckv, w=None, w_batch=0, wvec=[None] * B)
    # ---- weights: ("vec", n_w[, w_batch]) or ("table", lengths per row, w_row or None, w_ld)
    wspec = c.get("weights")
    if wspec and wspec[0] == "vec":
        n_w = wspec[1]
        w_batch = wspec[2] if len(wspec) > 2 else B
        vec = torch.rand(n_w, generator=gen) * 1.5 + 0.25
        vec[0], vec[-1] = 0.3, 1.9                                   # far from 1: the window's ends are visible
        s.update(w=vec.float().to(DEV), n_w=n_w, w_ld=0, w_len=None, w_row=None, w_batch=w_batch, table=False)
        for b in range(w_batch):
            assert n_w <= Nk[b], (c["id"], b)
            s["wvec"][b] = vec.double()
    elif wspec:
        _, lens, w_row, w_ld = wspec
        R = len(lens)
        w_batch = len(w_row) if w_row is not None else min(B, R)
        tab = torch.full((R, w_ld), float("nan"))
        for r, n in enumerate(lens):
            if n:
                row = torch.rand(n, generator=gen) * 1.5 + 0.25
                row[0], row[-1] = 0.3, 1.9
                tab[r, :n] = row
        s.update(w=tab.float().to(DEV), n_w=0, w_ld=w_ld, w_len=torch.tensor(lens, dtype=torch.int32, device=DEV),
                 w_row=torch.tensor(w_row, dtype=torch.int32, device=DEV) if w_row is not None else None,
                 w_batch=w_batch, table=True, lens=lens, rows=w_row if w_row is not None else list(range(w_batch)))
        for b in range(w_batch):
            n = lens[s["rows"][b]]
            if n:
                assert n <= Nk[b], (c["id"], b)
                s["wvec"][b] = tab[s["rows"][b], :n].double()
    s["kv_len_t"] = torch.tensor(kv_len, dtype=torch.int32, device=DEV) if kv_len is not None else None
    s["kv_slot_t"] = torch.tensor(kv_slot, dtype=torch.int32, device=DEV) if kv_slot is not None else None
    # the samples checked in detail: probes, run alone; with slots, ones that read different slots
    cand = [0, B - 1, B // 2] + ([next((b for b in range(B) if s["wvec"][b] is not None and b not in (0, B - 1)), 0)]
                                 if s["w"] is not None else [])
    chosen, used = [], set()
    for b in cand:
        if b not in chosen and slot_of[b] not in used:
            chosen.append(b)
            used.add(slot_of[b])
    s["probed"] = chosen
    _plant_probes(s, gen)
    return s


def _probe_keys(s, b):
    """List positions (in [self ; cond]) of the probe keys of sample b."""
    n_self, Nk, L = s["n_self"], s["Nk"][b], s["n_self"] + s["S"]
    keys = {0, Nk - 1}
    if Nk < L:
        keys.add(Nk)                                                  # first masked key (a conditioning row past kv_len)
    for k in (63, 64, 127, 128):                                     # 64-key chunk boundaries of the concatenated list
        if k < Nk:
            keys.add(k)
    if s["S"] and n_self:
        for k in (n_self + 63, n_self + 64):                         # the wgmma kernel's chunk boundaries inside cond
            if k < Nk:
                keys.add(k)
    g0 = 16 * ((Nk - 1) // 16)
    keys.update(k for k in (g0 - 1, g0) if 0 <= k < Nk)               # 16-key group boundary before the last group
    if s["wvec"][b] is not None:
        keys.update((Nk - len(s["wvec"][b]), Nk - 1))                # first and last weighted keys
    return sorted(keys)


def _key_row(s, b, j):
    """(tensor, row, column offset of k, column offset of v) of list position j of sample b."""
    E = s["E"]
    if j < s["n_self"]:
        return s["qkv"], b * s["P"] + j, E, 2 * E
    return s["ckv"].view(-1, 2 * E), s["slot_of"][b] * s["S"] + j - s["n_self"], 0, E


def _plant_probes(s, gen):
    P, H, hd, E = s["P"], s["H"], s["hd"], s["E"]
    for b in reversed(s["probed"]):
        keys = _probe_keys(s, b)
        rows = [0, P - 1, P // 2, 1, P - 2, P // 3, 2 * P // 3]
        q = s["qkv"][b * P:(b + 1) * P, :E].double().view(P, H, hd)
        for n, j in enumerate(keys):
            i = rows[n % len(rows)] % P
            qi = q[i]                                                 # [H, hd]
            zmax = _row_zmax(s, b, i)                                 # [H]
            # 4 above the row's max; the first masked key 24 above, so that a kernel that lets it into the running max
            # (while keeping its P at 0) leaves every other P of the row an fp16 zero
            lift = 24.0 if j == s["Nk"][b] else 4.0
            alpha = (zmax + lift) * math.sqrt(hd) / (qi * qi).sum(-1).clamp_min(1e-6)
            t, r, ko, vo = _key_row(s, b, j)
            t[r, ko:ko + E] = (alpha[:, None] * qi).reshape(E).half()
            t[r, vo:vo + E] = ((torch.rand(H, hd, generator=gen) * 2 + 2) *
                               torch.sign(torch.randn(H, hd, generator=gen))).reshape(E).half().to(DEV)


def _row_zmax(s, b, i):
    k, _, _ = _keys(s, [b])
    P, H, hd, E = s["P"], s["H"], s["hd"], s["E"]
    q = s["qkv"][b * P + i, :E].double().view(H, 1, hd)
    z = (q * k[0]).sum(-1) / math.sqrt(hd)                            # [H, L]
    z[:, s["Nk"][b]:] = -math.inf
    return z.amax(-1).clamp_min(0.0)


def _keys(s, bs):
    """k, v [G, H, L, hd] fp64 (L = n_self + S, the padded [self ; cond] list) and q [G, H, P, hd] of samples bs."""
    P, H, hd, E, S = s["P"], s["H"], s["hd"], s["E"], s["S"]
    G = len(bs)
    idx = torch.tensor(bs, device=DEV)
    qs = s["qkv"].view(-1, P, 3 * E)[idx]
    kp, vp = [], []
    if s["n_self"]:
        kp.append(qs[..., E:2 * E])
        vp.append(qs[..., 2 * E:])
    if S:
        cc = s["ckv"][torch.tensor([s["slot_of"][b] for b in bs], device=DEV)]
        kp.append(cc[..., :E])
        vp.append(cc[..., E:])
    L = s["n_self"] + S
    k = torch.cat(kp, 1).double().view(G, L, H, hd).transpose(1, 2)
    v = torch.cat(vp, 1).double().view(G, L, H, hd).transpose(1, 2)
    q = qs[..., :E].double().view(G, P, H, hd).transpose(1, 2)
    return k, v, q


# ------------------------------------------------------------------ fp64 reference
def _ref64(s, bs, mutation=None, bound=True):
    """ref [G, H, P, hd] (and the bound) of samples bs, optionally of a mutated kernel:
    drop_last, first_masked, drop_group, shift_w, renorm."""
    k, v, q = _keys(s, bs)
    G, L, hd = len(bs), k.shape[2], s["hd"]
    pos = torch.arange(L, device=DEV)
    Nk = torch.tensor([s["Nk"][b] for b in bs], device=DEV)
    valid = pos[None, :] < Nk[:, None]
    w = torch.ones(G, L, dtype=torch.float64, device=DEV)
    for g, b in enumerate(bs):
        wv = s["wvec"][b]
        if wv is not None:
            n, nk = len(wv), s["Nk"][b]
            if mutation == "shift_w":             # the window one key earlier: [nk - n - 1, nk - 1)
                lo = nk - n - 1
                w[g, max(lo, 0):nk - 1] = wv.to(DEV)[max(0, -lo):]
            else:
                w[g, nk - n:nk] = wv.to(DEV)
    if mutation == "drop_last":
        valid[torch.arange(G), Nk - 1] = False
    elif mutation == "first_masked":
        valid = pos[None, :] < torch.clamp(Nk + 1, max=L)[:, None]
    elif mutation == "drop_group":
        valid = pos[None, :] < (16 * ((Nk - 1) // 16))[:, None]
    z = q @ k.transpose(-1, -2) / math.sqrt(hd)                       # [G, H, P, L]
    vm = valid[:, None, None, :]
    zm = z.masked_fill(~vm, -math.inf)
    zmax = zm.amax(-1, keepdim=True)
    e = torch.exp(zm - zmax.clamp_min(-1e300))
    p = e / e.sum(-1, keepdim=True)
    pt = p * w[:, None, None, :]
    if mutation == "renorm":
        pt = pt / pt.sum(-1, keepdim=True)
    ref = (pt @ v).nan_to_num(0.0)
    if not bound:
        return ref
    A = pt @ v.abs()
    qk = q.abs() @ k.abs().transpose(-1, -2) / math.sqrt(hd)
    lam = LOG2E * (z.abs() + zmax.abs() + qk).masked_fill(~vm, 0.0).amax(-1, keepdim=True)
    vmax = v.abs().masked_fill(~valid[:, None, :, None], 0.0).amax(-2, keepdim=True)
    sub = Nk.double()[:, None, None, None] * 2.0 ** -25 * vmax
    bnd = U16 * ref.abs() + TAU_P * A + TAU_S * lam * (A + ref.abs()) + sub
    return ref, bnd, dict(A=A, lam=lam, sub=sub)


def _groups(s, bs):
    per = s["H"] * s["P"] * (s["n_self"] + s["S"])
    G = max(1, (1 << 24) // per)
    return [bs[i:i + G] for i in range(0, len(bs), G)]


# ------------------------------------------------------------------ launch
class _Out:
    """out [B*P, E] fp16 inside a buffer with guard bands on both sides, all prefilled with a sentinel bit pattern."""

    def __init__(self, n, pre=136, post=72):
        self.n, self.pre = n, pre
        self.bits = torch.full((pre + n + post,), SENTINEL, dtype=torch.int16, device=DEV)

    def ptr(self):
        return self.bits.data_ptr() + 2 * self.pre

    def val(self):
        return self.bits[self.pre:self.pre + self.n].view(torch.float16)

    def check(self, what):
        g = torch.cat([self.bits[:self.pre], self.bits[self.pre + self.n:]])
        assert bool((g == SENTINEL).all()), f"{what}: {int((g != SENTINEL).sum())} guard elements changed"
        n_in = int((self.bits[self.pre:self.pre + self.n] == SENTINEL).sum())
        assert n_in == 0, f"{what}: {n_in} output elements never written"


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _call(s, out_ptr, **ov):
    """pb200_attention_slots on case s, with any argument overridden; returns the return code."""
    from paella_b200 import _lib
    a = dict(qkv=s["qkv"], ckv=s["ckv"], kv_len=s["kv_len_t"], kv_slot=s["kv_slot_t"], n_slots=s["n_slots"] if s["kv_slot"] else 0,
             B=s["B"], P=s["P"], S=s["S"], E=s["E"], H=s["H"], self_=int(bool(s["n_self"])), w=s["w"], n_w=s.get("n_w", 0),
             w_ld=s.get("w_ld", 0), w_len=s.get("w_len"), w_row=s.get("w_row"), w_batch=s["w_batch"])
    a.update(ov)
    rc = _lib.lib().pb200_attention_slots(_p(a["qkv"]), _p(a["ckv"]), _p(a["kv_len"]), _p(a["kv_slot"]), a["n_slots"], ctypes.c_void_p(out_ptr),
                                          a["B"], a["P"], a["S"], a["E"], a["H"], a["self_"], _p(a["w"]), a["n_w"], a["w_ld"],
                                          _p(a["w_len"]), _p(a["w_row"]), a["w_batch"], _lib.current_stream())
    torch.cuda.synchronize()
    return rc


def _run(s, **ov):
    from paella_b200 import _lib
    o = _Out(s["B"] * s["P"] * s["E"] if "B" not in ov else ov["B"] * s["P"] * s["E"])
    _lib.check(_call(s, o.ptr(), **ov), "pb200_attention_slots")
    o.check("attention")
    return o.val().clone().view(-1, s["E"])


def _sample(out, s, b):
    P, H, hd = s["P"], s["H"], s["hd"]
    return out[b * P:(b + 1) * P].view(P, H, hd).transpose(0, 1)     # [H, P, hd]


def _alone(s, b):
    """Sample b at B = 1 with its own copy of its slot and of its weight row."""
    P, S = s["P"], s["S"]
    slot = s["slot_of"][b]
    ov = dict(qkv=s["qkv"][b * P:(b + 1) * P].clone(), B=1, kv_slot=None, n_slots=0)
    if S:
        ov["ckv"] = s["ckv"][slot:slot + 1].clone()
        ov["kv_len"] = s["kv_len_t"][slot:slot + 1].clone() if s["kv_len_t"] is not None else None
    if s["w"] is not None:
        ov["w_batch"] = 1 if b < s["w_batch"] else 0
        if s["table"] and b < s["w_batch"]:
            r = s["rows"][b]
            ov.update(w=s["w"][r:r + 1].clone(), w_len=s["w_len"][r:r + 1].clone(), w_row=None)
    return _run(s, **ov)


# ------------------------------------------------------------------ isolation
def _poison_rows(s):
    """(ckv row mask, weight-table element mask) of what no sample may read."""
    cm = None
    if s["S"]:
        cm = torch.zeros(s["n_slots"], s["S"], dtype=torch.bool, device=DEV)
        used = set(s["slot_of"])
        for sl in range(s["n_slots"]):
            if sl not in used:
                cm[sl] = True
            elif s["kv_len"] is not None:
                cm[sl, s["kv_len"][sl]:] = True
    wm = None
    if s["w"] is not None and s["table"]:
        wm = torch.zeros_like(s["w"], dtype=torch.bool)
        used = set(s["rows"])
        for r in range(wm.shape[0]):
            wm[r, (s["lens"][r] if r in used else 0):] = True
    return cm, wm


def _poisoned(t, mask, kind):
    """A copy of t with the masked rows / elements NaN, or +Inf and -Inf alternating."""
    t = t.clone()
    x = t[mask]
    alt = torch.arange(x.numel(), device=DEV).view_as(x) % 2 == 0
    t[mask] = torch.full_like(x, float("nan")) if kind == "nan" else torch.where(alt, float("inf"), float("-inf")).to(t.dtype)
    return t


def _isolation(s, out):
    cm, wm = _poison_rows(s)
    checked = 0
    if (cm is not None and bool(cm.any())) or (wm is not None and bool(wm.any())):
        for kind in ("nan", "inf"):
            ov = {}
            if cm is not None and bool(cm.any()):
                ov["ckv"] = _poisoned(s["ckv"], cm, kind)
            if wm is not None and bool(wm.any()):
                ov["w"] = _poisoned(s["w"], wm, kind)
            got = _run(s, **ov)
            assert torch.equal(got, out), f"output changed with {kind} in rows no sample may read ({int((got != out).sum())} elements, " \
                                          f"{int(torch.isnan(got).sum())} NaN)"
            checked += 1
    if s["c"].get("isolate_qkv"):
        P = s["P"]
        for b in (1, s["B"] - 1):
            m = torch.ones(s["B"] * P, dtype=torch.bool, device=DEV)
            m[b * P:(b + 1) * P] = False
            for kind in ("nan", "inf"):
                got = _run(s, qkv=_poisoned(s["qkv"], m, kind))
                assert torch.equal(_sample(got, s, b), _sample(out, s, b)), \
                    f"sample {b} changed with {kind} in the other samples' qkv ({int(torch.isnan(_sample(got, s, b)).sum())} NaN)"
                checked += 1
    for b in s["probed"]:
        assert torch.equal(_sample(_alone(s, b), s, 0), _sample(out, s, b)), f"sample {b} differs from the same sample run alone"
    return checked


# ------------------------------------------------------------------ one case
MUTATIONS = ("drop_last", "first_masked", "drop_group", "shift_w", "renorm")


def _run_case(c, kernel):
    s = _make(c)
    out = _run(s)
    again = _run(s)
    assert torch.equal(out, again), "a second launch differs"
    assert bool(torch.isfinite(out.float()).all()), f"{int((~torch.isfinite(out.float())).sum())} non-finite outputs"
    B = s["B"]
    # calibration record: the TAU_P the errors would need with no TAU_S term, and the TAU_S they would need with no TAU_P term
    worst, tau_p_alone, tau_s_alone = 0.0, 0.0, 0.0
    for bs in _groups(s, list(range(B))):
        ref, bnd, parts = _ref64(s, bs)
        got = torch.stack([_sample(out, s, b) for b in bs]).double()
        err = (got - ref).abs()
        worst = max(worst, float((err / bnd).max()))
        base = err - U16 * ref.abs() - parts["sub"]
        tau_p_alone = max(tau_p_alone, float((base / parts["A"].clamp_min(1e-30)).max()))
        tau_s_alone = max(tau_s_alone, float((base / (parts["lam"] * (parts["A"] + ref.abs())).clamp_min(1e-30)).max()))
    # sensitivity on the probed samples
    bs = s["probed"]
    ref, bnd, _ = _ref64(s, bs)
    sens = {}
    L = s["n_self"] + s["S"]
    for m in MUTATIONS:
        if m == "first_masked" and not any(s["Nk"][b] < L for b in bs):
            continue
        if m in ("shift_w", "renorm") and not any(s["wvec"][b] is not None for b in bs):
            continue
        mut = _ref64(s, bs, mutation=m, bound=False)
        sens[m] = float(((mut - ref).abs() / bnd).max())
    row = dict(kernel=kernel, case=c["id"], B=B, P=s["P"], H=s["H"], hd=s["hd"], S=s["S"], err_over_bound=worst,
               tau_p_alone=tau_p_alone, tau_s_alone=tau_s_alone, big_logits=c.get("logits") == "big",
               sensitivity=min(sens.values()), sens=sens)
    row["isolation_variants"] = _isolation(s, out)
    # shared slots == each sample with its own copy; all-equal table == the vector; unweighted rows == the unweighted call
    if s["kv_slot"] is not None:
        own = _run(s, ckv=s["ckv"][torch.tensor(s["slot_of"], device=DEV)].contiguous(),
                   kv_len=s["kv_len_t"][s["kv_slot_t"].long()].contiguous() if s["kv_len_t"] is not None else None,
                   kv_slot=None, n_slots=0)
        assert torch.equal(own, out), "a shared slot differs from each sample owning a copy of it"
    if s["w"] is not None and not s["table"]:
        n_w = s["n_w"]
        tab = torch.full((max(s["w_batch"], 1), n_w + 3), float("nan"), device=DEV)
        tab[:, :n_w] = s["w"]
        got = _run(s, w=tab, n_w=0, w_ld=n_w + 3, w_len=torch.full((tab.shape[0],), n_w, dtype=torch.int32, device=DEV), w_row=None)
        assert torch.equal(got, out), "an all-equal weight table differs from the single vector"
    if s["w"] is not None:
        plain = [b for b in range(B) if s["wvec"][b] is None]
        if plain:
            un = _run(s, w=None, n_w=0, w_ld=0, w_len=None, w_row=None, w_batch=0)
            for b in plain:
                assert torch.equal(_sample(un, s, b), _sample(out, s, b)), f"unweighted sample {b} differs from the unweighted call"
    assert worst <= 1.0, f"error/bound {worst:.3g}"
    assert row["sensitivity"] >= SENS_MIN, f"the bound cannot see a wrong kernel: {sens}"
    return row


# ------------------------------------------------------------------ a batch whose qkv holds more than 2^31 elements
def _big_case(kernel):
    hd = 64 if kernel == "mma" else 80
    H = 1280 // hd
    c = dict(id=f"qkv-over-2^31-hd{hd}", name="big", B=2200, P=256, H=H, S=8, self=True, hd=hd, kv_len="half")
    assert c["B"] * c["P"] * 3 * H * hd > BIG_ELEMS
    return c


def _run_big(kernel):
    c = _big_case(kernel)
    B, P, H, hd, S = c["B"], c["P"], c["H"], c["hd"], c["S"]
    E = H * hd
    g = torch.Generator(device=DEV).manual_seed(7)
    qkv = torch.randn(B * P, 3 * E, device=DEV, generator=g, dtype=torch.float16).mul_(1.5)
    ckv = (torch.randn(B, S, 2 * E, device=DEV, generator=g) * 1.5).half()
    kv_len = torch.randint(1, S + 1, (B,), device=DEV, generator=g, dtype=torch.int32)
    s = dict(c=c, B=B, P=P, H=H, S=S, hd=hd, E=E, n_self=P, n_slots=B, kv_slot=None, slot_of=list(range(B)),
             kv_len=kv_len.tolist(), qkv=qkv, ckv=ckv, w=None, w_batch=0, wvec=[None] * B, kv_len_t=kv_len, kv_slot_t=None)
    s["n_cond"] = s["kv_len"]
    s["Nk"] = [P + n for n in s["kv_len"]]
    out = _run(s)
    bs = [0, B // 2, B - 1]
    ref, bnd, _ = _ref64(s, bs)
    got = torch.stack([_sample(out, s, b) for b in bs]).double()
    ratio = float(((got - ref).abs() / bnd).max())
    s["probed"] = bs
    for b in bs:
        assert torch.equal(_sample(_alone(s, b), s, 0), _sample(out, s, b)), f"sample {b} differs from the same sample run alone"
    row = dict(kernel=kernel, case=c["id"], B=B, P=P, H=H, hd=hd, S=S, err_over_bound=ratio, qkv_elements=B * P * 3 * E)
    del qkv, out
    torch.cuda.empty_cache()
    assert ratio <= 1.0, f"error/bound {ratio:.3g}"
    return row


# ------------------------------------------------------------------ drivers
def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "attention" in e.name})


def _which_kernel_runs_hd80():
    s = _make(dict(_cases("wgmma")[0]))
    return _kernel_names(lambda: _run(s))


def _child_main():
    """Runs in a PB200_ATTN_MMA_SYNC=1 child: which kernel head_dim 80 runs, then every head_dim-80 case."""
    print("KERNELS", json.dumps(_which_kernel_runs_hd80()), flush=True)
    todo = [(c["id"], lambda c=c: _run_case(c, "mma80")) for c in _cases("mma80")]
    todo.append((_big_case("mma80")["id"], lambda: _run_big("mma80")))
    for cid, fn in todo:
        try:
            row = fn()
            _log(row)
            print("RES", json.dumps({"id": cid, "ok": True, "row": row}), flush=True)
        except Exception as e:          # report and go on: one case's failure must not hide the others
            print("RES", json.dumps({"id": cid, "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


_CHILD = {}


def _child_results():
    if not _CHILD:
        code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_attention_matrix as t; t._child_main()" % (ROOT, HERE)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                           env=dict(os.environ, PB200_ATTN_MMA_SYNC="1"))
        res = {"rc": r.returncode, "stderr": r.stderr[-3000:], "kernels": None, "cases": {}}
        for line in r.stdout.splitlines():
            if line.startswith("KERNELS "):
                res["kernels"] = json.loads(line[8:])
            elif line.startswith("RES "):
                j = json.loads(line[4:])
                res["cases"][j["id"]] = j
        _CHILD.update(res)
    return _CHILD


def test_head_dim_80_kernel_choice():
    """head_dim 80 runs the wgmma kernel by default and the mma.sync kernel under PB200_ATTN_MMA_SYNC=1."""
    names = _which_kernel_runs_hd80()
    assert names and all("wgmma" in n for n in names), names
    res = _child_results()
    assert res["kernels"] is not None, res["stderr"]
    assert res["kernels"] and all("attention_kernel<80>" in n for n in res["kernels"]), res["kernels"]
    assert res["rc"] == 0, res["stderr"]


def test_mma_sync_kernel_on_every_head_dim_80_case():
    """PB200_ATTN_MMA_SYNC=1 (child process) sends every head_dim-80 case, the wgmma kernel's shapes among them, to the
    mma.sync kernel, and all of them pass: the second kernel stays covered on the shapes the first one normally takes."""
    res = _child_results()
    want = [c["id"] for c in _cases("mma80")] + [_big_case("mma80")["id"]]
    missing = [cid for cid in want if cid not in res["cases"]]
    assert not missing, f"cases did not report (child rc {res['rc']}): {missing[:5]} {res['stderr']}"
    failed = {cid: res["cases"][cid]["msg"] for cid in want if not res["cases"][cid]["ok"]}
    assert not failed, failed
    assert res["rc"] == 0, res["stderr"]


@pytest.mark.parametrize("kernel,case", [(k, c["id"]) for k in KERNELS for c in _cases(k)]
                         + [(k, _big_case(k)["id"]) for k in KERNELS])
def test_attention_case(kernel, case):
    if kernel == "mma80":
        res = _child_results()
        got = res["cases"].get(case)
        assert got is not None, f"case did not report (child rc {res['rc']}): {res['stderr']}"
        assert got["ok"], got["msg"]
        return
    if case.startswith("qkv-over-2^31"):
        _log(_run_big(kernel))
        return
    c = next(c for c in _cases(kernel) if c["id"] == case)
    _log(_run_case(c, kernel))


@pytest.mark.parametrize("hd", [80, 16])
def test_refusals_leave_the_output_untouched(hd):
    """Unsupported head dims and E % nhead != 0 are errors; B = 0 and P = 0 are no-ops.  None of them writes the output."""
    from paella_b200 import _lib
    base = _make(dict(_cases("wgmma" if hd == 80 else "mma")[0]))
    H, P = 2, 16
    g = torch.Generator(device=DEV).manual_seed(3)

    def case(hd_, H_, B, P_, E=None):
        E = E or H_ * hd_
        s = dict(base, B=max(B, 1), P=max(P_, 1), H=H_, hd=hd_, E=E, S=8, n_self=max(P_, 1), kv_slot=None, kv_slot_t=None, w=None,
                 w_batch=0, kv_len_t=None)
        s["qkv"] = torch.randn(max(B, 1) * max(P_, 1), 3 * E, device=DEV, generator=g).half()
        s["ckv"] = torch.randn(max(B, 1), 8, 2 * E, device=DEV, generator=g).half()
        return s, dict(B=B, P=P_)

    for (hd_, H_, B, P_, E, want_err) in [(48, H, 2, P, None, True), (128, H, 2, P, None, True), (hd, 5, 2, P, 5 * hd + 8, True),
                                         (hd, H, 0, P, None, False), (hd, H, 2, 0, None, False)]:
        s, dims = case(hd_, H_, B, P_, E)
        o = _Out(max(B, 1) * max(P_, 1) * s["E"])
        before = o.bits.clone()
        rc = _call(s, o.ptr(), **dims)
        msg = _lib.lib().pb200_last_error()
        assert (rc != 0) == want_err, (hd_, H_, B, P_, E, rc, msg)
        assert torch.equal(o.bits, before), f"refused / empty call wrote the output (hd {hd_}, H {H_}, B {B}, P {P_})"
    assert torch.equal(_run(base), _run(base)), "the library is unusable after a refusal"
