"""Confidence-guided renoising without a GPU: argument validation (ops.confidence_table, utils.sample*, SamplingEngine.submit) before
any generator advances, the tau table's encoding, oracle/confidence.py against the reference fixture, the engine's step table, the
C ABI declarations, the ptxas reports of the two new kernels, and the SASS of every kernel that existed before them."""
import ctypes
import hashlib
import json
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ the tau table
def test_table_encoding():
    from paella_b200 import ops
    assert ops.confidence_table(None, 3) is None
    assert ops.confidence_table([None, None], 2) is None
    assert ops.confidence_table(0, 2).tolist() == [0.0, 0.0]
    assert ops.confidence_table(2.5, 3).tolist() == [2.5] * 3
    tab = ops.confidence_table([None, 0.0, 1, None, 3.25], 5)
    assert tab.dtype == torch.float32 and tab.device.type == "cpu"
    assert tab.tolist() == [-1.0, 0.0, 1.0, -1.0, 3.25]
    assert ops.confidence_table((None, 2.0), 2).tolist() == [-1.0, 2.0]
    assert ops.confidence_table(1.0, 1, 32768) is not None


@pytest.mark.parametrize("bad", [[1.0], [1.0, 1.0, 1.0], True, [None, False], -0.5, [None, -1.0], float("nan"), float("inf"),
                                 [None, float("-inf")], "1.0", [None, "2"], [None, [1.0]]])
def test_table_rejects(bad):
    from paella_b200 import ops
    with pytest.raises(ValueError):
        ops.confidence_table(bad, 2)


def test_table_rejects_a_grid_too_large_for_the_selection():
    from paella_b200 import ops
    with pytest.raises(ValueError, match="32768"):
        ops.confidence_table(1.0, 2, 32769)
    assert ops.confidence_table(None, 2, 10 ** 6) is None       # no entry, no bound


class _Stop(Exception):
    pass


class _Model:
    """Just enough of Paella for _sample_core's validation; any device work raises _Stop."""
    num_labels, n_attn_blocks = 64, 4

    def _device(self):
        return torch.device("cpu")

    def pag_default_blocks(self):
        return [1]

    def __getattr__(self, name):
        raise _Stop(name)


@pytest.mark.parametrize("kw,match", [
    (dict(confidence_renoise=[1.0]), "entries"),
    (dict(confidence_renoise=[None, True]), "choice temperature"),
    (dict(confidence_renoise=-1.0), "choice temperature"),
    (dict(confidence_renoise=[math.nan, None]), "choice temperature"),
    (dict(confidence_renoise=0.0, exact=True), "exact"),
    (dict(confidence_renoise=0.0, latent_shape=(2, 200, 200)), "32768"),
])
def test_sample_rejects_before_any_generator_advances(kw, match, monkeypatch):
    from paella_b200 import ops
    from paella_b200 import utils as U
    taken = []
    monkeypatch.setattr(ops, "randint", lambda *a, **k: taken.append("randint") or (_ for _ in ()).throw(_Stop()))
    monkeypatch.setattr(ops, "take_philox", lambda *a, **k: taken.append("philox") or (_ for _ in ()).throw(_Stop()))
    monkeypatch.setattr(ops, "philox_values", lambda *a, **k: taken.append("philox") or (_ for _ in ()).throw(_Stop()))
    shape = kw.pop("latent_shape", (2, 8, 8))
    exact = kw.pop("exact", False)
    with pytest.raises(ValueError, match=match):
        U.sample(_Model(), {"byt5": torch.zeros(shape[0], 2, 4)}, shape, None, steps=2, renoise_steps=1, cfg=0, exact=exact, **kw)
    assert taken == []


def test_sample_without_entries_takes_the_plain_path(monkeypatch):
    """[None, None] is the call without the argument: no per-sample table is forced (sampling_schedule returns None)."""
    from paella_b200 import ops
    from paella_b200 import utils as U
    seen = []
    real = U.sampling_schedule
    monkeypatch.setattr(ops, "randint", lambda *a, **k: (_ for _ in ()).throw(_Stop()))
    monkeypatch.setattr(ops, "to_device_packed", lambda *a, **k: (_ for _ in ()).throw(_Stop()))

    def spy(*a, **k):
        seen.append(k.get("always"))
        return real(*a, **k)
    monkeypatch.setattr(U, "sampling_schedule", spy)
    for conf in (None, [None, None]):
        with pytest.raises(_Stop):
            U.sample(_Model(), {"byt5": torch.zeros(2, 2, 4)}, (2, 8, 8), None, steps=2, renoise_steps=1, cfg=0,
                     confidence_renoise=conf)
    with pytest.raises(_Stop):
        U.sample(_Model(), {"byt5": torch.zeros(2, 2, 4)}, (2, 8, 8), None, steps=2, renoise_steps=1, cfg=0,
                 confidence_renoise=[None, 1.0])
    assert seen == [False, False, True]


# ------------------------------------------------------------------ the oracle against the reference fixture
@pytest.fixture(scope="module")
def fixture():
    z = np.load(os.path.join(ROOT, "tests", "golden", "confidence_tiny.npz"))
    return {k: z[k] for k in z.files}


def _case(f, name):
    T, tau, t, use_region = f[f"{name}:params"].tolist()
    which = str(f[f"{name}:which"])
    logits = f[f"logits_{which}"]
    tokens = f["ties_tokens"] if which == "ties" else f["tokens"]
    return T, tau, t, bool(use_region), logits, tokens


CASES = ["cond_T1_tau0", "cond_T02_tau2", "cond_T3_tau2", "guided_T1_tau2", "guided_T02_tau0", "guided_T3_tau0_region",
         "cond_T1_tau2_region", "ties_tau0", "cond_t0", "guided_t1"]


def test_fixture_lists_every_case(fixture):
    assert [str(n) for n in fixture["names"]] == CASES


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_fixture(fixture, name):
    from oracle import confidence as oc
    from oracle import philox
    f = fixture
    T, tau, t, use_region, logits, tokens = _case(f, name)
    B, K, H, W = logits.shape
    u = philox.rand(B * H * W, int(f["seed"]), int(f["offset"]), int(f["sm_count"])).reshape(B, H, W)
    assert np.array_equal(u, f["u"])
    inv_t = np.float32(1.0) / np.float32(T)
    for b in range(B):
        lg = logits[b].reshape(K, H * W).T
        c = oc.token_logprob(lg, inv_t, tokens[b].reshape(-1))
        assert np.abs(c - f[f"{name}:logp"][b].reshape(-1)).max() < 1e-9
        region = f["region"][b].reshape(-1) if use_region else None
        m = oc.select(f[f"{name}:logp"][b].reshape(-1), u[b], tau, t, region)
        assert np.array_equal(m, f[f"{name}:mask"][b].reshape(-1)), name
        n_cand = int(region.sum()) if use_region else H * W
        assert int(m.sum()) == oc.renoise_count(t, n_cand)
        if use_region:
            assert not m[~region].any()


def test_oracle_ties_go_to_the_lowest_indices(fixture):
    from oracle import confidence as oc
    T, tau, t, _, logits, tokens = _case(fixture, "ties_tau0")
    c = fixture["ties_tau0:logp"][0].reshape(-1)
    m = fixture["ties_tau0:mask"][0].reshape(-1)
    k = oc.order_keys(oc.keys(c, fixture["u"][0].reshape(-1), tau, t))
    thr = k[m].max()
    eq = np.flatnonzero(k == thr)
    taken = eq[m[eq]]
    assert len(eq) > len(taken) > 0 and np.array_equal(taken, eq[:len(taken)])
    assert (k[~m] >= thr).all()


def test_oracle_edge_rules():
    from oracle import confidence as oc
    u = np.array([0.5, 0.0, 0.25, 0.9], dtype=np.float32)
    c = np.array([-1.0, -3.0, np.nan, -2.0])
    assert oc.select(c, u, 1.0, -0.5).sum() == 0                   # t < 0 keeps
    assert oc.select(c, u, 1.0, 1.0).all()                         # t = 1 renoises every candidate
    # tau t = 0: token 1's u = 0 gives 0 * -inf, a NaN key like token 2's; NaN keys rank lowest, ties to the lower index
    assert oc.select(c, u, 0.0, 0.25).tolist() == [False, True, False, False]
    assert oc.select(c, u, 0.0, 0.5).tolist() == [False, True, True, False]
    assert oc.select(c, u, 1.0, 0.25).tolist() == [False, False, True, False]   # tau t > 0: token 1's key is -inf, above NaN
    assert oc.select(c, u, -1.0, 0.3).tolist() == [False, True, True, False]    # tau < 0: u <= t
    assert oc.gumbel(np.float32(0.0)) == -np.inf
    k = oc.order_keys(np.array([-np.inf, -1.0, -0.0, 0.0, 1.0, np.inf, np.nan], dtype=np.float32))
    assert k[-1] == 0 and (np.diff(k[:-1].astype(np.int64)) > 0).all()


# ------------------------------------------------------------------ the engine's step table
def _request(slot, steps, tau=-1.0, renoise_steps=None):
    from paella_b200 import utils as U
    from paella_b200.engine import Request
    params, r = U.sampling_schedule(1, steps, (1.0, 0.3), U._cfg_schedule((4.0, 4.0), 1, steps), 1.0, 0.0, always=True)
    q = Request(steps, steps - 1 if renoise_steps is None else renoise_steps, steps, True, params[:, 0], r[:, 0], confidence=tau)
    q.slot, q.uncond_slot = slot, 100 + slot
    return q


def test_engine_step_table_carries_tau_per_row():
    from paella_b200.engine import build_step_plan, step_host_table
    qs = [_request(0, 4, 0.0), _request(1, 4), _request(2, 4, 2.5, renoise_steps=1), _request(3, 3, 1.0)]
    for step in range(3):
        for q in qs:
            q.k = step
        plan = build_step_plan(qs, 8)
        want = any(q.k < q.renoise_steps and q.confidence >= 0 for q in plan.order)
        assert plan.confident == want
        host, lay = step_host_table(plan, [0, 0] * len(qs), [0, 0] * len(qs))
        assert ("tau" in lay) == want
        if want:
            f32 = host[lay["f32"][1]:lay["f32"][1] + lay["f32"][2]].view(torch.float32)
            _, o, n = lay["tau"]
            assert f32[o:o + n].tolist() == [q.confidence for q in plan.order]
    # step 2: request 2 (renoise_steps 1) no longer renoises; requests 0 and 3 still do
    assert plan.confident


def test_engine_step_table_without_confidence_is_unchanged():
    from paella_b200.engine import build_step_plan, step_host_table
    qs = [_request(0, 3), _request(1, 3, 1.0, renoise_steps=0)]      # request 1 never renoises
    plan = build_step_plan(qs, 8)
    assert not plan.confident
    _, lay = step_host_table(plan, [0, 0] * 2, [0, 0] * 2)
    assert "tau" not in lay


# ------------------------------------------------------------------ C ABI
NEW = ["pb200_paella_token_logprob", "pb200_renoise_confidence", "pb200_renoise_confidence_per_sample"]


def test_new_symbols_are_declared_exported_and_mirrored():
    from paella_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "paella_b200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(rf"\b{name}\s*\(", src), name
        assert name in _lib.SIGNATURES, name
    if os.path.exists(_lib.LIB_PATH):
        lib = ctypes.CDLL(_lib.LIB_PATH)
        for name in NEW:
            assert hasattr(lib, name), name
    assert "#define PB200_ABI_VERSION 4 " in open(os.path.join(ROOT, "include", "paella_b200.h")).read()
    assert len(_lib.SIGNATURES["pb200_paella_token_logprob"][1]) == 11
    assert len(_lib.SIGNATURES["pb200_renoise_confidence"][1]) == 14
    assert len(_lib.SIGNATURES["pb200_renoise_confidence_per_sample"][1]) == 14


# ------------------------------------------------------------------ ptxas reports and SASS
def _ptxas(name):
    path = os.path.join(ROOT, "paella_b200", "csrc", "build", f"{name}.ptxas.log")
    if not os.path.exists(path):
        pytest.skip("build first: the ptxas report is written by the build")
    return open(path).read()


@pytest.mark.parametrize("unit,kernel", [("token_logprob", "token_logprob_kernel"), ("renoise", "renoise_confidence_kernel")])
def test_new_kernels_do_not_spill(unit, kernel):
    log = _ptxas(unit)
    assert kernel in log
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in log
    assert "C7510" not in log


def _sass_hashes(so):
    """SHA-1 per function of its instruction and encoding lines, whitespace collapsed: the code and its control bits, without the
    module headers cuobjdump prints between functions of different objects (they name the neighbouring source file)."""
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    got, fn, buf = {}, None, []
    for line in out.splitlines() + ["Function : <end>"]:
        m = re.search(r"Function : (\S+)", line)
        if m:
            if fn:
                got[fn] = hashlib.sha1("\n".join(buf).encode()).hexdigest()
            fn, buf = m.group(1), []
        elif fn and re.match(r"\s+/\*(?:[0-9a-f]{4,}| 0x[0-9a-f]{16} )\*/", line):
            buf.append(" ".join(line.split()))
    return got


def test_existing_kernels_keep_their_sass():
    """tests/golden/sass_before_confidence.json holds the hash (_sass_hashes) of every kernel of libpaella_b200.so built without
    confidence-guided renoising, with the nvcc release that built it.  Its two kernels live in libpaella_b200_confidence.so, which
    libpaella_b200.so links: libpaella_b200.so must hold exactly the kernels it held, each with the same SASS (token_score_kernel,
    whose body token_logprob_kernel shares, included), and the new library exactly the two new kernels."""
    so = os.path.join(ROOT, "paella_b200", "libpaella_b200.so")
    conf = os.path.join(ROOT, "paella_b200", "libpaella_b200_confidence.so")
    if shutil.which("cuobjdump") is None or shutil.which("nvcc") is None or not os.path.exists(so) or not os.path.exists(conf):
        pytest.skip("cuobjdump, nvcc or the built libraries are not available")
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_before_confidence.json")))
    ver = subprocess.run(["nvcc", "--version"], capture_output=True, text=True, check=True).stdout
    if want["nvcc"] not in ver:
        pytest.skip(f"the reference hashes come from nvcc {want['nvcc']}")
    got = _sass_hashes(so)
    changed = [k for k, h in want["functions"].items() if got.get(k) != h]
    assert not changed, changed[:5]
    assert sorted(got) == sorted(want["functions"])
    assert sorted(_sass_hashes(conf)) == sorted(
        ["_ZN2pb20token_logprob_kernelE14CUtensorMap_stS0_iiiiPKfPKlPf",
         "_ZN2pb25renoise_confidence_kernelEPKlS1_S1_PKhPKiPKfS7_S7_lNS_11TorchPhiloxEPKmPlSB_"])


def test_main_library_links_the_confidence_library():
    """libpaella_b200.so finds libpaella_b200_confidence.so next to itself (DT_NEEDED with a $ORIGIN run path), so loading the
    one library the package loads is enough."""
    so = os.path.join(ROOT, "paella_b200", "libpaella_b200.so")
    if shutil.which("readelf") is None or not os.path.exists(so):
        pytest.skip("readelf or the built library is not available")
    dyn = subprocess.run(["readelf", "-d", so], capture_output=True, text=True, check=True).stdout
    assert "[libpaella_b200_confidence.so]" in dyn and "[$ORIGIN]" in dyn


def test_confidence_library_is_hopper_native():
    """test_sass_lint.py's rules for libpaella_b200.so, on the kernels of libpaella_b200_confidence.so: the log-probability kernel
    runs warpgroup MMA (HGMMA) fed by TMA (UTMALDG), with no mma.sync, and no kernel wraps a single-thread region in an
    ELECT ... BRA.U.ANY loop."""
    conf = os.path.join(ROOT, "paella_b200", "libpaella_b200_confidence.so")
    if shutil.which("cuobjdump") is None or not os.path.exists(conf):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run(["cuobjdump", "-sass", conf], capture_output=True, text=True, check=True).stdout
    funcs, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            funcs[fn] = []
        elif fn:
            funcs[fn].append(line)
    lp = "\n".join(next(v for k, v in funcs.items() if "token_logprob_kernel" in k))
    assert "HGMMA" in lp and "UTMALDG" in lp and "HMMA" not in lp
    assert all("BRA.U.ANY" not in "\n".join(v) for v in funcs.values())
