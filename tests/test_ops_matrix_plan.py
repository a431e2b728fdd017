"""CPU checks of test_gpu_ops_matrix.py's case table: every kernel of ops.cu and blocks.cu that libpaella_b200.so holds
(tests/golden/sass_before_confidence.json lists them) is run by at least one case, the Python restatements of the
dispatchers pick the instances the table claims, and the entries exposed for testing are declared, exported and bound."""
import ctypes
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import test_gpu_ops_matrix as M  # noqa: E402

TEMPLATE_ARGS = {"5uint4": "uint4", "j": "uint32_t", "h": "uint8_t"}
TESTING_ENTRIES = ["pb200_embed_tokens", "pb200_ln_rows", "pb200_ln_patchify2", "pb200_film_table", "pb200_mix_cast_f16",
                   "pb200_mix_cast_rows_f16", "pb200_pad_cast_f16", "pb200_gather_cast_f16", "pb200_replicate_rows",
                   "pb200_regional_masks", "pb200_guidance_mix", "pb200_dwconv_ln_pairs"]


def _instance(mangled):
    """_ZN2pb16dwconv_ln_kernelILi10ELb0ELb1EEEv... -> dwconv_ln_kernel<10,0,1>."""
    m = re.match(r"_ZN2pb(\d+)", mangled)
    n = int(m.group(1))
    name, rest = mangled[m.end():m.end() + n], mangled[m.end() + n:]
    if not rest.startswith("I"):
        return name
    args, rest = [], rest[1:]
    while not rest.startswith("E"):
        lit = re.match(r"L[ib](\d+)E", rest)
        if lit:
            args.append(lit.group(1))
            rest = rest[lit.end():]
            continue
        key = next(k for k in TEMPLATE_ARGS if rest.startswith(k))
        args.append(TEMPLATE_ARGS[key])
        rest = rest[len(key):]
    return f"{name}<{','.join(args)}>"


def _source_kernels():
    names = set()
    for f in ("ops.cu", "blocks.cu"):
        src = open(os.path.join(ROOT, "paella_b200", "csrc", f)).read()
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\((?:[^()]|\([^()]*\))*\)\s+)?(\w+)\s*\(", src))
    return names


def test_every_kernel_of_ops_and_blocks_is_covered():
    names = _source_kernels()
    assert {"embed_tokens_kernel", "ln_rows_kernel", "dwconv3_ln_patch_kernel", "ln_affine_kernel", "regional_masks_kernel"} <= names
    assert set(M.OUT_OF_SCOPE) <= names
    sass = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_before_confidence.json")))["functions"]
    instances = {_instance(k) for k in sass if re.match(r"_ZN2pb\d+", k)}
    ours = {i for i in instances if i.split("<")[0] in names and i.split("<")[0] not in M.OUT_OF_SCOPE}
    assert len(ours) == 56
    missing = sorted(ours - set(M.COVERAGE))
    assert not missing, f"no case runs: {missing}"
    assert not set(M.COVERAGE) - instances, "the table names instances the library does not hold"


def test_dwconv_dispatch_restatement():
    k = M._dw_kernel
    assert k(640, 3, 16, False, False, "default") == "dwconv_ln_kernel<5,0,0>"              # c <= 640: warp kernel
    assert k(648, 3, 8, True, False, "default") == "dwconv3_ln_patch_kernel<1,320,0>"      # k = 3, c > 640, w >= 8: patch
    assert k(648, 3, 7, False, True, "default") == "dwconv_ln_kernel<10,0,1>"              # w < 8: warp
    assert k(1000, 5, 16, False, False, "default") == "dwconv_ln_kernel<10,0,0>"           # k != 3: warp
    assert k(2056, 3, 16, False, False, "default") == "dwconv3_ln_patch_kernel<0,640,0>"
    assert k(2056, 3, 16, False, False, "warp") == "dwconv_ln_kernel<20,0,0>"
    assert k(256, 3, 3, False, False, "patch") == "dwconv3_ln_patch_kernel<0,64,0>"        # 64 threads
    assert k(264, 3, 3, False, False, "patch") == "dwconv3_ln_patch_kernel<0,160,0>"       # 66 -> 96 threads
    assert k(640, 3, 3, True, True, "patch") == "dwconv3_ln_patch_kernel<1,160,1>"
    assert k(1280, 3, 8, False, False, "patch") == "dwconv3_ln_patch_kernel<0,320,0>"
    assert k(520, 5, 16, False, False, "patch") == "dwconv_ln_kernel<5,0,0>"               # the knob needs k = 3
    assert k(128, 7, 3, True, False, "default") == "dwconv_ln_kernel<1,1,0>"
    # the table exercises idle threads in the patch kernel (c/4 not a multiple of 32), h % 2 and w % 8 != 0
    patch = [c for c in M.DW_CASES if "patch" in k(c["c"], c["k"], c["w"], c["skip"], c["wrap"], "default")]
    assert any((c["c"] // 4) % 32 for c in patch) and any(c["h"] % 2 and c["w"] % 8 for c in patch)
    assert {c["k"] for c in M.DW_CASES} == {1, 3, 5, 7}
    assert any(c["wrap"] and min(c["h"], c["w"]) < c["k"] for c in M.DW_CASES)


def test_grn_rows_per_cta_rule():
    r = M._grn_rows_per_cta
    assert r(3, 7, 2048, M.SM_H100) == (7, 256)           # P < 16: P rows
    assert r(3, 64, 8, M.SM_H100) == (8, 32)              # tpb < 256; 16 rows leave SMs idle -> 8
    assert r(26, 100, 5120, M.SM_H100) == (16, 256)       # 7 * 26 * 3 = 546 CTAs >= 4 * 132
    assert r(66, 64, 2056, M.SM_H100) == (16, 256)        # 4 * 66 * 2 = 528
    assert r(65, 64, 2056, M.SM_H100) == (8, 256)         # 520 < 528
    rpc = {r(c["b"], c["p"], c["n"], M.SM_H100)[0] for c in M.GRN_CASES}
    assert {16, 8}.issubset(rpc) and any(x < 8 for x in rpc)
    assert {c["n"] for c in M.GRN_CASES} == {8, 2048, 2056, 5120}
    assert {1, 7, 8, 15, 16, 17, 64, 100} <= {c["p"] for c in M.GRN_CASES}
    assert M._grn32_grid(7, 36) == 1 and M._grn32_grid(512, 8192) == 1024 and 512 * 8192 // 2048 > 1024


def test_other_dispatch_restatements():
    assert M._film_kernel(64) == "film_table_kernel<64>" and M._film_kernel(65) == "film_table_generic_kernel"
    assert {c["b"] for c in M.FILM_CASES} >= {1, 64, 65, 200} and any(c["t"] % 128 for c in M.FILM_CASES)
    assert M._replicate_kernel(48) == "replicate_rows_kernel<uint4>"
    assert M._replicate_kernel(36) == "replicate_rows_kernel<uint32_t>"
    assert M._replicate_kernel(37) == "replicate_rows_kernel<uint8_t>"
    assert M._layernorm_kernel(36, 1e-6, False, False) == "ln_rows_kernel<0>"
    assert M._layernorm_kernel(5, 1e-6, False, False) == "ln_affine_kernel"
    assert M._layernorm_kernel(36, 1e-5, False, False) == "ln_affine_kernel"
    assert M._layernorm_kernel(36, 1e-6, True, False) == "ln_affine_kernel"
    # embed: scalar and vector stores, ps 1 / 2 / 4, the 3072-element (48 KB) limit
    rl = {c["c"] * c["ps"] ** 2 for c in M.EMBED_CASES}
    assert 3072 in rl and any(x % 8 for x in rl) and any(x % 8 == 0 for x in rl)
    assert {c["ps"] for c in M.EMBED_CASES} == {1, 2, 4}
    # ln_rows: C / 4 not a multiple of 32, rows % 8 != 0
    assert {c["c"] for c in M.LN_CASES} == {4, 36, 260, 1284} and all(c["rows"] % 8 for c in M.LN_CASES)
    # casts: every n % 4, OP 3 with a sample boundary inside a thread's four elements
    assert {c["n"] % 4 for c in M.CAST_CASES} == {0, 1, 2, 3}
    assert all(M.CAST_PER[n] % 4 for n in M.CAST_PER)


def test_testing_entries_are_declared_exported_and_bound():
    from paella_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "paella_b200.h")).read()
    for name in TESTING_ENTRIES:
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES, name
    assert os.path.exists(_lib.LIB_PATH), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert all(hasattr(lib, n) for n in TESTING_ENTRIES)
    assert _lib.lib().pb200_abi_version() == 4
