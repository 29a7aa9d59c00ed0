"""The C-ABI library loads and exports every symbol include/f2nerf_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "f2nerf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(f2b_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_path():
    syms = declared_symbols()
    for need in ("f2b_sampler_count", "f2b_sampler_fill", "f2b_hash_fwd", "f2b_hash_bwd", "f2b_mlp_fwd", "f2b_mlp_bwd",
                 "f2b_composite_fwd", "f2b_composite_act_bwd", "f2b_early_stop_rays", "f2b_compact_slots", "f2b_sh_encode"):
        assert need in syms


def test_library_exports_every_declared_symbol():
    from f2nerf_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in include/f2nerf_b200.h but not exported: {missing}"


def test_header_declares_every_exported_symbol():
    """An f2b_ entry point the library exports but the header does not declare is reachable by no binding."""
    import subprocess
    from f2nerf_b200 import _lib
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {f[-1] for f in (line.split() for line in out.splitlines()) if f and f[-1].startswith("f2b_")}
    undeclared = sorted(exported - set(declared_symbols()))
    assert exported and not undeclared, f"exported but not declared in include/f2nerf_b200.h: {undeclared}"


def test_python_binding_covers_the_header():
    from f2nerf_b200 import _lib
    unbound = [s for s in declared_symbols() if s not in _lib.SIGNATURES and s != "f2b_last_error"]
    assert not unbound, f"no ctypes signature for: {unbound}"


def test_abi_version_and_error_string():
    from f2nerf_b200 import _lib
    assert _lib.lib.f2b_abi_version() == 1
    assert isinstance(_lib.lib.f2b_last_error(), bytes)


def test_no_product_import_of_the_oracle():
    """The product package must never reach into oracle/ (parity claims are void otherwise)."""
    pkg = os.path.join(ROOT, "f2nerf_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle_lib" not in txt and "libf2oracle" not in txt and "f2_oracle" not in txt, f


def test_table_grad_buffer_reuse_rules():
    """Renderer._table_grad_buffer (host logic, no GPU): the table-gradient storage is reused across steps — a NEW tensor object on
    the same storage each time, so autograd can take it as .grad without a copy — only while no tensor on last step's gradient is
    alive; a trainer that keeps .grad gets a fresh, fully zeroed tensor; the dead tail is zero in every case."""
    import torch
    from f2nerf_b200.renderer import Renderer, slab_groups
    r = Renderer.__new__(Renderer)
    a = r._table_grad_buffer((64, 2), "cpu")
    assert r._table_grad_tail_zero and float(a.abs().sum()) == 0.0 and a._use_count() == 1
    a[:34] += 1.0                                                  # "live prefix" written by a backward
    ptr = a.data_ptr()
    p = torch.nn.Parameter(torch.zeros(64, 2))
    p.grad = a
    del a
    b = r._table_grad_buffer((64, 2), "cpu")                       # last step's gradient is still held by the trainer
    assert b.data_ptr() != ptr and float(b.abs().sum()) == 0.0 and float(p.grad[:34].sum()) == 68.0
    p.grad = None
    del b
    c = r._table_grad_buffer((64, 2), "cpu")                       # released: the storage comes back, as a new tensor object
    assert c._use_count() == 1 and r._table_grad_tail_zero and float(c[34:].abs().sum()) == 0.0
    d = r._table_grad_buffer((32, 2), "cpu")                       # another shape: never a view of the old storage
    assert d.shape == (32, 2) and float(d.abs().sum()) == 0.0
    assert slab_groups() == ((12, 4), (8, 4), (4, 4), (0, 4))


def test_renderer_refuses_other_mlp_depths():
    """The launch sequences are built for the shipped field 32->64->16 and shader 32->64->64->16 only: a Renderer over other
    depths is refused at construction (the stand-alone operators keep both depths)."""
    import pytest
    from f2nerf_b200 import GlobalDataPool, Hash3DAnchored, Renderer, SHShader
    gdp = GlobalDataPool()
    for field_layers, shader_layers in ((2, 2), (1, 1)):
        field = Hash3DAnchored(gdp, log2_table_size=8, n_hidden_layers=field_layers, device="cpu")
        shader = SHShader(gdp, n_hiddens=shader_layers, device="cpu")
        with pytest.raises(NotImplementedError, match="MLP shapes"):
            Renderer(gdp, None, field, shader, n_images=2, device="cpu")
    Renderer(gdp, None, Hash3DAnchored(gdp, log2_table_size=8, device="cpu"), SHShader(gdp, device="cpu"), n_images=2, device="cpu")
