"""Top-k / top-p truncation without a device: argument validation and the host table (ops.truncation_table), the fp64 oracle
against a plain torch sort / cumsum formulation, exact=True with truncation, and SamplingEngine's per-step table layout."""
import random

import numpy as np
import pytest
import torch

from oracle.truncation import kept_set, truncated_winner
from paella_b200 import ops
from paella_b200 import utils as U
from paella_b200.engine import Request, build_step_plan, step_host_table

NL = 512


# ------------------------------------------------------------------ validation and the table
@pytest.mark.parametrize("top_k,top_p", [
    (-1, None), (2.0, None), (True, None), ("3", None), (torch.tensor([1.0, 2.0]), None), (torch.tensor([1, -1]), None),
    (torch.tensor([1, 2, 3]), None), (None, 0.0), (None, -0.5), (None, 1.5), (None, float("nan")), (None, True),
    (None, torch.tensor([0.5, 0.0])), (None, torch.tensor([0.5, float("nan")])), (None, torch.tensor([1, 1])),
    (None, torch.tensor([0.5])),
])
def test_bad_arguments_raise(top_k, top_p):
    with pytest.raises(ValueError):
        ops.truncation_table(top_k, top_p, 2, NL)


def test_cuda_tensor_is_refused():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA tensor")
    with pytest.raises(ValueError):
        ops.truncation_table(torch.tensor([1, 2], device="cuda"), None, 2, NL)


def test_off_rows_give_no_table():
    assert ops.truncation_table(None, None, 3, NL) is None
    assert ops.truncation_table(0, 1.0, 3, NL) is None
    assert ops.truncation_table(NL, 1, 3, NL) is None                     # k >= num_labels keeps every code
    assert ops.truncation_table(torch.tensor([0, NL + 5, NL]), torch.tensor([1.0, 1.0, 1.0]), 3, NL) is None


def test_table_scalars_and_per_sample_mixes():
    k, p = ops.truncation_table(64, None, 3, NL)
    assert k.dtype == torch.int32 and p.dtype == torch.float32
    assert k.tolist() == [64] * 3 and p.tolist() == [1.0] * 3
    k, p = ops.truncation_table(None, 0.9, 2, NL)
    assert k.tolist() == [0, 0] and p.tolist() == [np.float32(0.9)] * 2
    k, p = ops.truncation_table(torch.tensor([0, 7, NL, 1], dtype=torch.int64), torch.tensor([1.0, 0.5, 0.99, 1.0], dtype=torch.float64),
                                4, NL)
    assert k.tolist() == [0, 7, 0, 1]
    assert p.tolist() == [1.0, 0.5, np.float32(0.99), 1.0]


def test_exact_with_truncation_raises_before_any_work():
    # exact=True is checked before the model is touched: a stand-in model that fails on any device use
    class NoDevice:
        num_labels = NL

        def _device(self):
            return torch.device("cpu")

    with pytest.raises(ValueError, match="exact=True"):
        U._sample_core(NoDevice(), {}, (1, 2, 2), None, None, 2, 1, (1.0, 0.2), None, 1.0, 0.0, 2, "multinomial", None, True,
                       False, top_k=5)


# ------------------------------------------------------------------ the oracle against torch sort / cumsum
def _torch_kept(s: torch.Tensor, k: int, p: float) -> torch.Tensor:
    s = s.double()
    keep = torch.ones_like(s, dtype=torch.bool)
    if 0 < k < s.numel():
        keep = s >= torch.sort(s, descending=True).values[k - 1]
    if 0 < p < 1:
        w = torch.where(keep, torch.exp(s - s.max()), torch.zeros_like(s))
        sv, idx = torch.sort(s, descending=True)
        cum = torch.cumsum(w[idx], 0)
        first = int(torch.nonzero(cum >= p * w.sum())[0])          # the first position reaching the mass: its value is tau_p
        keep &= s >= sv[first]
    return keep


def _row(rng, n, ties):
    s = rng.standard_normal(n) * 3.0
    if ties:      # planted ties: a few values repeated across the row, including the top
        vals = np.sort(s)[::-1][:5]
        for v in vals:
            s[rng.choice(n, 3, replace=False)] = v
    return s


@pytest.mark.parametrize("ties", [False, True])
def test_oracle_matches_sort_cumsum(ties):
    rng = np.random.default_rng(5 if ties else 6)
    n = 300
    for trial in range(60):
        s = _row(rng, n, ties)
        order = np.sort(s)[::-1]
        ks = [0, 1, 7, n - 1, n, n + 3]
        # p near a cumulative boundary: just either side of one prefix's mass fraction (1e-9 apart, far above the fp64
        # rounding of the two formulations' differently ordered sums)
        w = np.exp(order - order[0])
        frac = np.cumsum(w) / w.sum()
        j = int(rng.integers(0, n - 1))
        ps = [1.0, 0.5, 0.9, 0.99, frac[j] * (1 - 1e-9), min(1.0, frac[j] * (1 + 1e-9))]
        for k in ks:
            for p in ps:
                if not 0 < p <= 1:
                    continue
                want = _torch_kept(torch.from_numpy(s), k, float(p)).numpy()
                got = kept_set(s, k, float(p))
                assert np.array_equal(got, want), (trial, k, p)
                if k == 1:
                    assert got.sum() == (s == s.max()).sum()
                if k >= n and p == 1.0:
                    assert got.all()


def test_oracle_winner_is_gumbel_max_over_the_kept_set():
    rng = np.random.default_rng(9)
    s = rng.standard_normal((20, 64))
    q = rng.exponential(1.0, (20, 64))
    full = (s - np.log(q)).argmax(1)
    assert np.array_equal(truncated_winner(s, q), full)
    top1 = truncated_winner(s, q, k=1)
    assert np.array_equal(top1, s.argmax(1))
    for k, p in ((7, 1.0), (0, 0.5), (7, 0.9)):
        win = truncated_winner(s, q, k, p)
        keep = kept_set(s, k, p)
        assert keep[np.arange(20), win].all()


# ------------------------------------------------------------------ the engine's per-step table
def _request(rng, slot, steps, top_k, top_p, mode="multinomial"):
    cfg = rng.choice([None, (8.0, 8.0)])
    cfgs = U._cfg_schedule(cfg, 1, steps)
    params, r = U.sampling_schedule(1, steps, (0.7, 0.3), cfgs, 1.0, 0.0, always=True)
    q = Request(steps, steps - 1, steps, cfg is not None, params[:, 0], r[:, 0], mode=mode, top_k=top_k, top_p=top_p)
    q.slot, q.uncond_slot = slot, 99
    return q


def test_step_table_layout_with_and_without_truncation():
    rng = random.Random(4)
    for trial in range(40):
        reqs = []
        for j in range(rng.randint(1, 9)):
            tk = rng.choice([0, 0, 1, 64])
            tp = rng.choice([1.0, 1.0, 0.9])
            reqs.append(_request(rng, j, rng.choice([1, 2, 4]), tk, tp, rng.choice(["multinomial", "multinomial", "argmax"])))
        active = list(reqs)
        while active:
            plan = build_step_plan(active)
            Bc = len(plan.order)
            want_tr = any(dr and (q.top_k > 0 or q.top_p < 1.0) for q, dr in zip(plan.order, plan.draws))
            assert plan.truncates == want_tr
            draw = [0, 0] * Bc
            renoise = [0, 0] * Bc
            host, lay = step_host_table(plan, draw, renoise)
            f32 = host[lay["f32"][1]:lay["f32"][1] + lay["f32"][2]].view(torch.float32)
            i32 = host[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32)

            def part(name):
                dt, o, n = lay[name]
                return (f32 if dt == "f32" else i32)[o:o + n]
            assert torch.equal(part("r"), plan.r) and torch.equal(part("params"), plan.params.view(-1))
            assert torch.equal(part("row_slot"), plan.row_slot) and torch.equal(part("kv_slot"), plan.kv_slot)
            if want_tr:
                assert part("top_k").tolist() == [q.top_k for q in plan.order]
                assert torch.equal(part("top_p"), torch.tensor([q.top_p for q in plan.order], dtype=torch.float32))
            else:        # no row truncates: the table is the one of a step without truncation
                assert "top_k" not in lay and "top_p" not in lay
                assert host.numel() == 4 * Bc + (5 * Bc + 1) // 2 + (2 * Bc + plan.n_pairs + lay["modes"][2] + 1) // 2
            for q in plan.order:
                q.k += 1
            active = [q for q in active if q.k < q.steps]
