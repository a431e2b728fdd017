"""CPU-side checks of the drop-in boundary: the shared library loads without a GPU and exports exactly the
entry points include/paella_b200.h declares; the ctypes table mirrors the header; the product never imports
the oracle; no compute call is made here."""
import ctypes
import inspect
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "paella_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pb200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from paella_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _header_functions()
    assert len(names) >= 35
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/paella_b200.h but not exported"


def test_ctypes_table_mirrors_header():
    from paella_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _header_functions()
    l = _lib.lib()
    assert l.pb200_abi_version() == 4
    assert l.pb200_last_error() is not None


def test_plan_consumes_reference_state_dict_names():
    """Host-only: the C plan's parameter list == the reference's state-dict keys (golden tiny config)."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from helpers import load_golden
    from paella_b200 import _lib
    cfg, sd, _ = load_golden("paella_tiny.npz")
    L = _lib.lib()
    c = _lib.PaellaConfig()
    for k in ("c_in", "c_out", "num_labels", "c_r", "patch_size", "c_cond", "clip_embd", "byt5_embd", "clip_seq_len", "kernel_size"):
        setattr(c, k, int(cfg[k]))
    c.self_attn, c.n_levels = 1, len(cfg["c_hidden"])
    for i in range(c.n_levels):
        c.c_hidden[i], c.nhead[i], c.blocks[i] = cfg["c_hidden"][i], cfg["nhead"][i], cfg["blocks"][i]
        c.level_config[i].value = cfg["level_config"][i].encode()
    h = ctypes.c_void_p()
    _lib.check(L.pb200_paella_create(ctypes.byref(c), ctypes.byref(h)), "create")
    names = {L.pb200_paella_param_name(h, i).decode(): L.pb200_paella_param_numel(h, i) for i in range(L.pb200_paella_num_params(h))}
    assert set(names) == set(sd)
    assert all(names[k] == sd[k].numel() for k in sd)
    L.pb200_paella_destroy(h)
    vcfg, vsd, _ = load_golden("vqgan_tiny.npz")
    vc = _lib.VqganConfig(vcfg["levels"], vcfg["bottleneck_blocks"], vcfg["c_hidden"], vcfg["c_latent"], vcfg["codebook_size"], 0.3764)
    vh = ctypes.c_void_p()
    _lib.check(L.pb200_vqgan_create(ctypes.byref(vc), ctypes.byref(vh)), "vq create")
    vnames = {L.pb200_vqgan_param_name(vh, i).decode(): L.pb200_vqgan_param_numel(vh, i) for i in range(L.pb200_vqgan_num_params(vh))}
    want = {k for k in vsd if not k.endswith("num_batches_tracked")}
    assert set(vnames) == want
    assert all(vnames[k] == vsd[k].numel() for k in want)
    L.pb200_vqgan_destroy(vh)


def test_python_mirror_has_reference_surface():
    import inspect
    from paella_b200 import modules, utils, vqgan
    sig = inspect.signature(modules.Paella.__init__)
    assert list(sig.parameters)[1:] == ["c_in", "c_out", "num_labels", "c_r", "patch_size", "c_cond", "c_hidden", "nhead", "blocks",
                                        "level_config", "clip_embd", "byt5_embd", "clip_seq_len", "kernel_size", "dropout", "self_attn"]
    assert list(inspect.signature(modules.Paella.forward).parameters)[1:7] == ["x", "r", "byt5", "clip", "clip_image", "x_cat"]
    assert list(inspect.signature(utils.sample).parameters)[:11] == ["model", "model_inputs", "latent_shape", "unconditional_inputs",
                                                                     "steps", "renoise_steps", "temperature", "cfg", "t_start", "t_end", "device"]
    assert list(inspect.signature(vqgan.VQModel.__init__).parameters)[1:] == ["levels", "bottleneck_blocks", "c_hidden", "c_latent",
                                                                              "codebook_size", "scale_factor"]
    for name in ("Attention2D", "LayerNorm2d", "GlobalResponseNorm", "ResBlock", "AttnBlock", "FeedForwardBlock", "TimestepBlock"):
        assert hasattr(modules, name)
    # notebook import paths
    import importlib
    for mod in ("src.vqgan", "utils.modules", "utils.alter_attention", "src.utils", "src.modules"):
        importlib.import_module(mod)


def test_load_conditional_models_reads_reference_checkpoint_layout(tmp_path):
    """ref/src/utils.py:24-32: `{'state_dict': ...}` VQGAN checkpoint -> eval-mode VQModel with those weights."""
    import torch
    from paella_b200 import utils, vqgan
    src = vqgan.VQModel()
    with torch.no_grad():
        for p in src.parameters():
            p.add_(0.01)
    path = str(tmp_path / "vqgan_f4.pt")
    torch.save({"state_dict": src.state_dict()}, path)
    assert list(inspect.signature(utils.load_conditional_models).parameters) == ["byt5_model_name", "vqgan_path", "device"]
    vq, byt5 = utils.load_conditional_models(None, path, "cpu")
    assert byt5 is None and not vq.training and not any(p.requires_grad for p in vq.parameters())
    for k, v in src.state_dict().items():
        assert torch.equal(vq.state_dict()[k], v), k
    import src.utils as shim
    assert shim.load_conditional_models is utils.load_conditional_models


def test_gemm_tile_plan_on_a_148_sm_part():
    """Host-side tile planner on a part with more SMs than the H100 (pure arithmetic, no device work): the bench
    workload's GEMM shapes keep their 256-wide one-CTA tiles, and small problems still get narrow tiles."""
    import ctypes
    from paella_b200 import _lib
    L = _lib.lib()

    def plan(m, n, k, sms=148):
        bn = ctypes.c_int()
        _lib.check(L.pb200_gemm_plan(m, n, k, sms, ctypes.byref(bn)), "gemm_plan")
        return bn.value
    assert plan(8192, 1280, 5120) == 256
    assert plan(8192, 1280, 1280) == 256
    assert plan(8192, 5120, 1280) == 256
    assert plan(8192, 3840, 1280) == 256
    assert plan(64, 1280, 1280) == 64
    assert plan(300, 640, 64) == 64


def test_gemm_tile_plan_on_a_132_sm_part():
    """Host-side tile planner (pure arithmetic, no device work): the BLOCK_N the bench workload's GEMM shapes get on a
    132-SM H100 (DESIGN.md section 3).  Every tile is one CTA's and BLOCK_N wide on sm_90a."""
    import ctypes
    from paella_b200 import _lib
    L = _lib.lib()

    def plan(m, n, k, sms=132):
        bn = ctypes.c_int()
        _lib.check(L.pb200_gemm_plan(m, n, k, sms, ctypes.byref(bn)), "gemm_plan")
        return bn.value
    # level-1 MLP GEMMs, out-projection and QKV projection: 256-wide tiles
    assert plan(8192, 1280, 5120) == 256
    assert plan(8192, 1280, 1280) == 256
    assert plan(8192, 5120, 1280) == 256
    assert plan(8192, 3840, 1280) == 256
    # a single 128-row tile with a short N: narrow tiles spread it over more SMs
    assert plan(64, 1280, 1280) == 64
    # every answer is a legal configuration, on any SM count
    for sms in (148, 132, 66):
        for m, n, k in [(8192, 1280, 5120), (300, 640, 64), (32768, 2560, 640), (2048, 1280, 1280), (12032, 512, 256)]:
            assert plan(m, n, k, sms) in (64, 128, 256)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "paella_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f"{f} imports the oracle"


def test_cpu_tensors_raise_not_fallback():
    import torch
    from paella_b200 import _lib, ops
    with pytest.raises(_lib.PaellaB200Error):
        ops.vq_nearest(torch.zeros(4, 4), torch.zeros(8, 4))
    # the stand-alone building blocks go through the same boundary
    from paella_b200.modules import LayerNorm2d, ResBlock
    with pytest.raises(_lib.PaellaB200Error):
        ResBlock(32)(torch.zeros(1, 32, 4, 4))
    with pytest.raises(_lib.PaellaB200Error):
        LayerNorm2d(32)(torch.zeros(1, 32, 4, 4))
