"""The C-ABI library loads and exports every symbol include/b200_paged_attn.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

from nanovllm import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200_paged_attn.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def test_library_built():
    assert nat.lib_path().exists(), "run `make -C nano-vllm_b200/csrc` (or __graft_entry__.build())"


def test_exports_match_header():
    names = declared_symbols()
    assert len(names) >= 17
    lib = ctypes.CDLL(str(nat.lib_path()))
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    assert set(nat.SIGNATURES) == set(names), "ctypes table and header disagree"


def test_plain_flavour_exports_the_same_abi():
    """`make NOPDL=1` (the same sources without programmatic dependent launch) must stay a drop-in for the default library."""
    pdl = nat.lib_path().with_name("libb200attn_nopdl.so")
    if not pdl.exists():
        pytest.skip("plain flavour not built (make -C nano-vllm_b200/csrc NOPDL=1)")
    lib = ctypes.CDLL(str(pdl))
    for n in declared_symbols():
        assert hasattr(lib, n), f"{n} missing from the plain flavour"
    assert lib.b200_abi_version() == 2


def test_host_only_entry_points():
    lib = nat.load()
    assert lib.b200_abi_version() == 2
    assert lib.b200_strerror(0) == b"ok"
    assert b"not bound" in lib.b200_strerror(-4)
    assert lib.b200_sm_count(None) == 0
    assert lib.b200_decode_workspace_bytes(None, 4, 4) == 0
    # the per-thread PDL switch returns the previous setting (enabled by default) and is idempotent
    assert lib.b200_set_pdl(0) == 1 and lib.b200_set_pdl(0) == 0
    assert lib.b200_set_pdl(1) == 0 and lib.b200_set_pdl(1) == 1


def test_no_cpu_fallback(monkeypatch):
    """Without a CUDA device the product refuses to run instead of falling back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    nat.reset_handle()
    with pytest.raises(nat.B200Error):
        nat.handle()
    from nanovllm import ops
    with pytest.raises(nat.B200Error):
        ops.silu_mul(torch.zeros(2, 16, dtype=torch.bfloat16))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "nano-vllm_b200", "nanovllm")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports the oracle"


def _header_prototypes():
    """name -> (return type, [parameter declarations]) parsed from the header."""
    text = open(os.path.join(ROOT, "include", "b200_paged_attn.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"([A-Za-z_][\w\s\*]*?)\b(b200_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        ret, name, params = m.group(1).strip(), m.group(2), m.group(3).strip()
        plist = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
        protos[name] = (ret, plist)
    return protos


def _ctype_of(decl: str):
    if "*" in decl:
        return "ptr"
    for c_name, kind in (("int64_t", ctypes.c_int64), ("uint64_t", ctypes.c_uint64), ("size_t", ctypes.c_size_t),
                         ("float", ctypes.c_float), ("int", ctypes.c_int)):
        if re.search(rf"\b{c_name}\b", decl):
            return kind
    raise AssertionError(f"unrecognised C type in {decl!r}")


def test_ctypes_table_matches_header_prototypes():
    """Every argument of every entry point has the width and kind the header declares (a drifted table would corrupt
    arguments silently)."""
    protos = _header_prototypes()
    assert set(protos) == set(nat.SIGNATURES)
    for name, (ret, params) in protos.items():
        restype, argtypes = nat.SIGNATURES[name]
        assert len(argtypes) == len(params), f"{name}: {len(argtypes)} ctypes arguments, header declares {len(params)}"
        for i, (decl, at) in enumerate(zip(params, argtypes)):
            want = _ctype_of(decl)
            if want == "ptr":
                assert at is ctypes.c_void_p or issubclass(at, ctypes._Pointer), f"{name} arg {i} ({decl}): {at}"
            else:
                assert at is want, f"{name} arg {i} ({decl}): table says {at}, header says {want}"
        if "*" in ret:
            assert restype in (ctypes.c_char_p, ctypes.c_void_p), name
        elif ret == "void":
            assert restype is None, name
        else:
            assert restype is _ctype_of(ret), f"{name}: return {ret} vs {restype}"


def test_integration_doc_binding_matches_table():
    """The ctypes stub INTEGRATION.md shows a maintainer is the same binding the product uses."""
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    text = re.sub(r"\n\s+(?=_)", " ", text)                       # join continued argtypes lines
    short = {"_vp": ctypes.c_void_p, "_i": ctypes.c_int, "_i64": ctypes.c_int64, "_f": ctypes.c_float, "_sz": ctypes.c_size_t}
    seen = 0
    for m in re.finditer(r"_lib\.(b200_\w+)\.argtypes = \[([^\]]*)\]", text):
        name, args = m.group(1), [a.strip() for a in m.group(2).split(",") if a.strip()]
        want = nat.SIGNATURES[name][1]
        assert len(args) == len(want), name
        for a, w in zip(args, want):
            if a in short:
                assert short[a] is w, f"{name}: {a} vs {w}"
            else:
                assert "POINTER" in a and issubclass(w, ctypes._Pointer), f"{name}: {a} vs {w}"
        seen += 1
    assert seen >= 5


def test_argument_validation_needs_no_gpu():
    """Entry points reject bad arguments before touching CUDA (error behaviour is part of the ABI)."""
    lib = nat.load()
    EINVAL, EUNSUPPORTED = -1, -2
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16          # 16-byte aligned scratch address
    assert lib.b200_silu_mul(None, p, 1, 8, None) == EINVAL
    assert lib.b200_silu_mul(p, p, 1, 12, None) == EINVAL               # inter must be a multiple of 8
    assert lib.b200_silu_mul(p + 2, p, 1, 8, None) == EINVAL            # misaligned
    assert lib.b200_silu_mul(p, p, 0, 8, None) == 0                     # empty batch: nothing to do
    assert lib.b200_embedding(None, p, p, 1, 8, 16, None) == EINVAL
    assert lib.b200_gather_tokens(p, None, p, 1, None) == EINVAL
    assert lib.b200_gather_tokens(p, p, p, 0, None) == 0
    assert lib.b200_kv_bind(None, p, p, 1, 1, 16, 1, 128) == EINVAL
    # tensor-parallel exchange: world in [2, 8], rank inside it, row length a multiple of 8 and at most 8192
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, p, p, 0, 1, p, p, p, 1, 1024, 1e-6, None) == EINVAL
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, p, p, 2, 2, p, p, p, 1, 1024, 1e-6, None) == EINVAL
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, p, p, 0, 2, p, p, p, 1, 1001, 1e-6, None) == EUNSUPPORTED
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, p, p, 0, 2, p, p, p, 0, 1024, 1e-6, None) == 0
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, p, p, 0, 2, p, p, p, 1, 8200, 1e-6, None) == EUNSUPPORTED
    assert lib.b200_allreduce_add_rmsnorm(p, 8, 0, p, p, p, 0, 2, p, p, p, 1, 1024, 1e-6, None) == EUNSUPPORTED  # data 16 B
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 2, p, p, p, 0, 2, p, p, p, 1, 1024, 1e-6, None) == EUNSUPPORTED  # flags 4 B
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, p, p, -1, 2, p, p, p, 1, 1024, 1e-6, None) == EINVAL
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, None, p, p, 0, 2, p, p, p, 1, 1024, 1e-6, None) == EINVAL   # no epoch
    assert lib.b200_allreduce_add_rmsnorm(p, 0, 0, p, None, p, 0, 2, p, p, p, 1, 1024, 1e-6, None) == EINVAL   # no done
    assert lib.b200_allreduce_add_rmsnorm_nvls(p, None, 0, 0, p, p, p, 0, 2, p, p, p, 1, 1024, 1e-6, None) == EINVAL
    assert lib.b200_allreduce_add_rmsnorm_nvls(p, p, 0, 0, p, p, p, 0, 9, p, p, p, 1, 1024, 1e-6, None) == EINVAL
    assert lib.b200_allreduce_add_rmsnorm_nvls(p, p, 0, 0, p, p, p, 0, 2, p, p, p, 0, 1024, 1e-6, None) == 0
    # wgmma linear layer: k a multiple of 64, split-K only with the partial-sum epilogue, block sizes from the list
    assert lib.b200_linear(None, 64, p, p, 64, 1, 64, 64, 0, 32, 1, 0, None) == EINVAL
    assert lib.b200_linear(p, 64, p, p, 64, 1, 64, 96, 0, 32, 1, 0, None) == EUNSUPPORTED
    assert lib.b200_linear(p, 128, p, p, 64, 1, 64, 128, 0, 32, 2, 0, None) == EINVAL
    assert lib.b200_linear(p, 64, p, p, 64, 1, 48, 64, 0, 32, 1, 0, None) == EUNSUPPORTED
    assert lib.b200_linear(p, 64, p, p, 64, 0, 64, 64, 0, 32, 1, 0, None) == 0
    # fused LM head + sampling: hidden, head, key workspace and one of out / out_keys are required
    assert lib.b200_lm_head_sample(None, 64, p, 1, 128, 64, None, 0, 0, 0, None, p, p, None, 128, 0, None) == EINVAL
    assert lib.b200_lm_head_sample(p, 64, p, 1, 128, 64, None, 0, 0, 0, None, p, None, None, 128, 0, None) == EINVAL
    assert lib.b200_lm_head_sample(p, 64, p, 1, 128, 72, None, 0, 0, 0, None, p, p, None, 128, 0, None) == EUNSUPPORTED
    assert lib.b200_lm_head_sample(p, 64, p, 1, 128, 64, None, 2 ** 32, 0, 0, None, p, p, None, 128, 0, None) == EUNSUPPORTED
    assert lib.b200_lm_head_sample(p, 64, p, 0, 128, 64, None, 0, 0, 0, None, p, p, None, 128, 0, None) == 0
    assert lib.b200_lm_head_sample(p, 64, p, 1, 128, 64, None, 0, 0, 0, None, p, p, None, 0, 0, None) == EUNSUPPORTED
    assert lib.b200_add_rmsnorm_partials(None, 1, p, p, p, 1, 64, 1e-6, 0, None) == EINVAL
    assert lib.b200_add_rmsnorm_partials(p, 1, p, p, p, 1, 10000, 1e-6, 0, None) == EUNSUPPORTED
