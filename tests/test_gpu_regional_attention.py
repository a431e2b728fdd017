"""Both attention kernels with regional prompts (pb200_attention_regional) against an fp64 reference with per-query masks.

A query of a sample b < mask_batch sees every self key and, in one softmax, the conditioning rows of each prompt whose bit is set
in its mask byte: prompt 0 is the sample's kv_slot, prompts 1..R the slots of its region_slot row (mask_row picks the row).  Each
case runs the wgmma kernel (head_dim 80), the mma.sync kernel (16, 32, 64, 96) or the mma.sync kernel at head_dim 80 (a
PB200_ATTN_MMA_SYNC=1 child process, as in test_gpu_attention_matrix.py), at ragged query counts and prompts of 0 to 129 rows,
with overlapping masks, a slot shared by two samples' prompts, a permuted mask_row and an unmasked unconditional sample, and checks:
  * every element within test_gpu_attention_matrix's error bound of the fp64 result, in its guard-banded sentinel buffer;
  * the bound can see a wrong kernel: probe keys on the first and last row of a prompt make dropping that prompt for a query
    that sees it, or reading it for one that does not, move some element by SENS_MIN times its bound;
  * isolation, bit for bit: new finite K/V in a slot leave every query that sees no prompt in that slot unchanged; NaN, then
    +-Inf, in the slot of a prompt no query of a tile sees leave that tile unchanged (the tile loads no chunk of it);
  * a sample whose masks are all bit 0, and the unconditional sample, give the plain kernel's output bit for bit.
"""
import ctypes
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_attention_matrix import LOG2E, SENS_MIN, TAU_P, TAU_S, U16, _Out

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
P_VALUES = (1, 16, 63, 64, 65, 256)
LENS = (0, 1, 63, 64, 65, 129, 17, 40)          # kv_len of the 8 cache slots, rotated per case
B, MASK_BATCH, R = 3, 2, 3
KV_SLOT = (6, 7, 6)                             # sample 2 (unmasked) shares sample 0's prompt-0 slot
REGION_SLOT = ((0, 1, 2), (3, 4, 5), (5, -1, 2))  # rows; slot 5 and 2 appear in two rows
MASK_ROW = (2, 0)


def _cases(kernel):
    hds = {"wgmma": (80,), "mma80": (80,), "mma": (16, 32, 64, 96)}[kernel]
    return [dict(id=f"{kernel}-hd{hd}-P{P}", hd=hd, P=P, rot=i) for hd in hds for i, P in enumerate(P_VALUES)]


def _make(c, seed=0):
    g = torch.Generator(device=DEV).manual_seed(1000 * c["P"] + c["hd"] + seed)
    hd, P = c["hd"], c["P"]
    H = 2
    E = H * hd
    lens = [LENS[(j + c["rot"]) % len(LENS)] for j in range(8)]
    S = max(max(lens), 1)
    s = dict(c, H=H, E=E, S=S, lens=lens)
    s["qkv"] = (torch.randn(B * P, 3 * E, device=DEV, generator=g) * 0.5).half()
    s["ckv"] = (torch.randn(8, S, 2 * E, device=DEV, generator=g) * 0.5).half()
    s["kv_len"] = torch.tensor(lens, dtype=torch.int32, device=DEV)
    s["kv_slot"] = torch.tensor(KV_SLOT, dtype=torch.int32, device=DEV)
    s["region_slot"] = torch.tensor(REGION_SLOT, dtype=torch.int32, device=DEV)
    s["mask_row"] = torch.tensor(MASK_ROW, dtype=torch.int32, device=DEV)
    # overlapping random masks over the prompts that exist in the sample's row; bit 0 where nothing else is set
    m = torch.zeros(MASK_BATCH, P, dtype=torch.uint8)
    cg = torch.Generator().manual_seed(c["P"] + 7 * c["hd"] + seed)
    for b in range(MASK_BATCH):
        row = REGION_SLOT[MASK_ROW[b]]
        for k in range(1, R + 1):
            if row[k - 1] >= 0:
                m[b] |= (torch.rand(P, generator=cg) < 0.4).to(torch.uint8) << k
        m[b] |= (torch.rand(P, generator=cg) < 0.3).to(torch.uint8)
        m[b][m[b] == 0] = 1
    s["q_mask"] = m.to(DEV)
    return s


def _prompts(s, b):
    """[(bit, slot)] of sample b's prompts."""
    out = [(0, KV_SLOT[b])]
    if b < MASK_BATCH:
        out += [(k, sl) for k, sl in enumerate(REGION_SLOT[MASK_ROW[b]], start=1) if sl >= 0]
    return out


def _ref64(s, b, vis_override=None):
    """fp64 result [H, P, hd] of sample b and its bound, keys = [self ; every prompt's rows], masked per query."""
    P, E, H, hd = s["P"], s["E"], s["H"], s["hd"]
    qkv = s["qkv"][b * P:(b + 1) * P].double()
    q = qkv[:, :E].view(P, H, hd).transpose(0, 1)
    ks, vs, vis = [qkv[:, E:2 * E]], [qkv[:, 2 * E:]], [torch.ones(P, P, dtype=torch.bool, device=DEV)]
    mask = s["q_mask"][b].long() if b < MASK_BATCH else torch.ones(P, dtype=torch.long, device=DEV)
    for bit, sl in _prompts(s, b):
        n = s["lens"][sl]
        kv = s["ckv"][sl, :n].double()
        ks.append(kv[:, :E]); vs.append(kv[:, E:])
        vis.append(((mask >> bit) & 1).bool()[:, None].expand(P, n))
    k = torch.cat(ks).view(-1, H, hd).transpose(0, 1)
    v = torch.cat(vs).view(-1, H, hd).transpose(0, 1)
    vm = torch.cat(vis, 1)
    if vis_override is not None:
        vm = vis_override(vm)
    z = q @ k.transpose(-1, -2) / math.sqrt(hd)
    zm = z.masked_fill(~vm[None], -math.inf)
    zmax = zm.amax(-1, keepdim=True)
    p = torch.exp(zm - zmax) / torch.exp(zm - zmax).sum(-1, keepdim=True)
    ref = p @ v
    A = p @ v.abs()
    qk = q.abs() @ k.abs().transpose(-1, -2) / math.sqrt(hd)
    lam = LOG2E * (z.abs() + zmax.abs() + qk).masked_fill(~vm[None], 0.0).amax(-1, keepdim=True)
    vmax = (v.abs()[:, None] * vm[None, :, :, None]).amax(-2)
    sub = vm.sum(-1).double()[None, :, None] * 2.0 ** -25 * vmax
    return ref, U16 * ref.abs() + TAU_P * A + TAU_S * lam * (A + ref.abs()) + sub, vm


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _run(s, regional=True):
    from paella_b200 import _lib
    P, E = s["P"], s["E"]
    o = _Out(B * P * E)
    L = _lib.lib()
    args = (_p(s["qkv"]), _p(s["ckv"]), _p(s["kv_len"]), _p(s["kv_slot"]), 8, ctypes.c_void_p(o.ptr()), B, P, s["S"], E, s["H"], 1,
            None, 0, 0, None, None, 0)
    if regional:
        rc = L.pb200_attention_regional(*args, _p(s["q_mask"]), _p(s["region_slot"]), _p(s["mask_row"]), R, MASK_BATCH,
                                        _lib.current_stream())
    else:
        rc = L.pb200_attention_slots(*args, _lib.current_stream())
    assert rc == 0, L.pb200_last_error()
    torch.cuda.synchronize()
    o.check("regional attention" if regional else "plain attention")
    return o.val().view(B, P, s["H"], s["hd"]).transpose(1, 2).clone()


def _plant(s, b, bit, rows):
    """Probe keys on the first and last row of sample b's prompt `bit`: k = alpha q_i for query rows[0] / rows[1], large v."""
    sl = dict(_prompts(s, b))[bit]
    n = s["lens"][sl]
    if n == 0:
        return None
    P, E, hd, H = s["P"], s["E"], s["hd"], s["H"]
    for j, i in ((0, rows[0]), (n - 1, rows[1])):
        q = s["qkv"][b * P + i, :E].float().view(H, hd)
        kk = q * (6.0 * math.sqrt(hd) / q.pow(2).sum(-1, keepdim=True).clamp_min(1e-3))
        s["ckv"][sl, j, :E] = kk.reshape(-1).half()
        s["ckv"][sl, j, E:] = 4.0
    return sl, n


def _sensitivity(s):
    """min over probes of max |ref_mutated - ref| / bound: dropping a seen prompt / reading an unseen one, for sample 0."""
    P = s["P"]
    m = s["q_mask"][0].long()
    sens = []
    for bit, _ in _prompts(s, 0)[1:]:
        seen = ((m >> bit) & 1).nonzero().flatten().tolist()
        unseen = ((~m >> bit) & 1).nonzero().flatten().tolist()
        for rows, drop in ((seen, True), (unseen, False)):
            if not rows:
                continue
            r2 = [rows[0], rows[-1]]
            if _plant(s, 0, bit, r2) is None:
                continue
            ref, bnd, _ = _ref64(s, 0)
            lo = P + sum(s["lens"][sl] for kb, sl in _prompts(s, 0) if kb < bit)
            hi = lo + s["lens"][dict(_prompts(s, 0))[bit]]

            def flip(vm, r2=r2, lo=lo, hi=hi, drop=drop):
                vm = vm.clone()
                for i in r2:
                    vm[i, lo:hi] = not drop
                return vm
            mut, _, _ = _ref64(s, 0, flip)
            sens.append(float(((mut - ref).abs() / bnd).amax()))
    return min(sens) if sens else float("inf")


def _run_case(c):
    s = _make(c)
    got = _run(s)
    worst = 0.0
    for b in range(B):
        ref, bnd, _ = _ref64(s, b)
        err = (got[b].double() - ref).abs() / bnd
        worst = max(worst, float(err.amax()))
    assert worst <= 1.0, f"{c['id']}: error / bound {worst:.3f}"
    assert torch.equal(_run(s).view(torch.int16), got.view(torch.int16)), "second launch differs"
    plain = _run(s, regional=False)
    assert torch.equal(got[2].view(torch.int16), plain[2].view(torch.int16)), "the unmasked sample differs from the plain kernel"
    # a sample whose masks are all bit 0 is the plain kernel's, bit for bit
    s0 = dict(s, q_mask=s["q_mask"].clone())
    s0["q_mask"][1] = 1
    assert torch.equal(_run(s0)[1].view(torch.int16), plain[1].view(torch.int16)), "an all-bit-0 sample differs from the plain kernel"
    # isolation: new finite K/V in slot 0 (prompt 1 of sample 1 alone) leave every query that does not see it unchanged
    seen1 = ((s["q_mask"][1].long() >> 1) & 1).bool()
    s1 = dict(s, ckv=s["ckv"].clone())
    s1["ckv"][0] = (torch.randn_like(s1["ckv"][0].float()) * 0.5).half()
    got1 = _run(s1)
    assert torch.equal(got1[1][:, ~seen1].view(torch.int16), got[1][:, ~seen1].view(torch.int16)), "a query read a prompt it does not see"
    assert torch.equal(got1[0].view(torch.int16), got[0].view(torch.int16)) and torch.equal(got1[2].view(torch.int16), got[2].view(torch.int16))
    # chunk skip: no query of sample 1's last tile sees prompt 1 (slot 0); NaN then +-Inf there leave that tile unchanged
    t0 = ((s["P"] - 1) // 64) * 64
    s2 = dict(s, q_mask=s["q_mask"].clone())
    s2["q_mask"][1, t0:] &= 0xFD
    s2["q_mask"][1][s2["q_mask"][1] == 0] = 1
    base = _run(s2)
    for val in (float("nan"), float("inf"), float("-inf")):
        s3 = dict(s2, ckv=s2["ckv"].clone())
        s3["ckv"][0] = val
        out = _run(s3)
        assert torch.equal(out[1][:, t0:].view(torch.int16), base[1][:, t0:].view(torch.int16)), f"a tile read an unseen prompt ({val})"
    sens = _sensitivity(s)
    assert sens >= SENS_MIN, f"{c['id']}: sensitivity {sens:.1f} < {SENS_MIN}"
    return {"id": c["id"], "err_over_bound": worst, "sensitivity": sens}


def _child_main():
    for c in _cases("mma80"):
        try:
            print("RES", json.dumps({"id": c["id"], "ok": True, "row": _run_case(c)}), flush=True)
        except Exception as e:          # report and go on: one case's failure must not hide the others
            print("RES", json.dumps({"id": c["id"], "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


_CHILD = {}


def _child_results():
    if not _CHILD:
        code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_regional_attention as t; t._child_main()" % (ROOT, HERE)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, PB200_ATTN_MMA_SYNC="1"))
        _CHILD.update(rc=r.returncode, stderr=r.stderr[-3000:], cases={})
        for line in r.stdout.splitlines():
            if line.startswith("RES "):
                j = json.loads(line[4:])
                _CHILD["cases"][j["id"]] = j
    return _CHILD


@pytest.mark.parametrize("kernel,case", [(k, c["id"]) for k in ("wgmma", "mma80", "mma") for c in _cases(k)])
def test_regional_attention_case(kernel, case):
    from helpers import log_jsonl
    if kernel == "mma80":
        res = _child_results()
        got = res["cases"].get(case)
        assert got is not None, f"case did not report (child rc {res['rc']}): {res['stderr']}"
        assert got["ok"], got["msg"]
        return
    log_jsonl("regional_attention.jsonl", _run_case(next(c for c in _cases(kernel) if c["id"] == case)))


def test_regional_attention_refusals():
    """More than 7 regions, or a mask batch past the batch, is an error that leaves the output untouched."""
    from paella_b200 import _lib
    s = _make(_cases("wgmma")[0])
    P, E = s["P"], s["E"]
    for max_regions, mask_batch in ((8, MASK_BATCH), (R, B + 1), (-1, MASK_BATCH)):
        o = _Out(B * P * E)
        before = o.bits.clone()
        rc = _lib.lib().pb200_attention_regional(_p(s["qkv"]), _p(s["ckv"]), _p(s["kv_len"]), _p(s["kv_slot"]), 8, ctypes.c_void_p(o.ptr()),
                                                 B, P, s["S"], E, s["H"], 1, None, 0, 0, None, None, 0, _p(s["q_mask"]),
                                                 _p(s["region_slot"]), _p(s["mask_row"]), max_regions, mask_batch, _lib.current_stream())
        torch.cuda.synchronize()
        assert rc != 0 and torch.equal(o.bits, before)
