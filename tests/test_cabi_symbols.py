"""CPU: the C-ABI library builds, loads, and exports every symbol include/b2m.h declares; without a GPU the
product refuses to run (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b2m.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2m_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound(lib_built):
    from moe_infinity_b200 import _lib
    lib = _lib.load()
    declared = _declared()
    assert len(declared) >= 25
    bound = {n for n, _, _ in _lib.SYMBOLS}
    for name in declared:
        assert hasattr(lib, name), f"libb2m.so does not export {name}"
        assert name in bound, f"{name} is declared in b2m.h but not bound in _lib.SYMBOLS"
    assert lib.b2m_version() == 1


def test_config_struct_layout_matches_header(lib_built):
    from moe_infinity_b200 import _lib
    # 18 int32 + float + int32 (80 B) + double + 5 int32 + float = 112 bytes with natural alignment
    assert C.sizeof(_lib.Config) == 112
    assert _lib.Config.device_memory_ratio.offset % 8 == 0


def test_library_has_hopper_sass(lib_built):
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    assert "HGMMA" in sass, "wgmma missing"
    assert "UTMALDG" in sass, "TMA loads missing"
    assert "SYNCS" in sass, "mbarrier waits missing"
    assert "sm_90a" in sass


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_gpu_fails_loudly(lib_built):
    from moe_infinity_b200 import _lib
    lib = _lib.load()
    cfg = _lib.Config()
    cfg.struct_size = C.sizeof(_lib.Config)
    cfg.num_layers, cfg.num_experts, cfg.hidden, cfg.inter, cfg.top_k, cfg.max_tokens = 1, 8, 128, 256, 2, 16
    cfg.expert_type = _lib.EXPERT_MIXTRAL
    h = C.c_void_p()
    rc = lib.b2m_ctx_create(C.byref(cfg), C.byref(h))
    assert rc == _lib.B2M_ECUDA
    assert b"no CPU fallback" in lib.b2m_last_error(None)
    with pytest.raises(RuntimeError):
        from moe_infinity_b200 import MoEEngine
        MoEEngine(num_layers=1, num_experts=8, hidden=128, inter=256, top_k=2)


def test_bad_config_rejected(lib_built):
    from moe_infinity_b200 import _lib
    lib = _lib.load()
    cfg = _lib.Config()
    cfg.struct_size = 8
    h = C.c_void_p()
    assert lib.b2m_ctx_create(C.byref(cfg), C.byref(h)) == _lib.B2M_EINVAL
    cfg.struct_size = C.sizeof(_lib.Config)
    cfg.dtype = _lib.DTYPE_FP8
    assert lib.b2m_ctx_create(C.byref(cfg), C.byref(h)) == _lib.B2M_EUNSUPPORTED
    assert lib.b2m_ctx_create(None, None) == _lib.B2M_EINVAL
