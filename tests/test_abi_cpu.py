"""The C-ABI library loads without a GPU and exports every symbol include/b200sd.h declares (no compute calls)."""

def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    ge.build()
    from b200sd import _lib
    names = _lib.declared_symbols()
    assert len(names) >= 17 and "b200sd_linear" in names and "b200sd_attention" in names and "b200sd_conv2d" in names
    lib = _lib.load()
    for n in names:
        assert hasattr(lib, n), n
    assert lib.b200sd_version().decode().endswith("sm_90a")


def test_missing_library_fails_loudly(tmp_path):
    from b200sd import _lib
    import pytest
    with pytest.raises(_lib.B200SDError):
        _lib.load(str(tmp_path / "libmissing.so"))


def test_engine_refuses_cpu_device():
    import pytest
    from b200sd import config as C, engine as E
    with pytest.raises(RuntimeError):
        E.SDEngine({}, C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP, device="cpu")


def test_every_entry_point_is_documented():
    """INTEGRATION.md's table names the upstream operation behind every exported symbol"""
    import os
    from b200sd import _lib
    doc = open(os.path.join(os.path.dirname(__file__), "..", "INTEGRATION.md")).read()
    for name in _lib.declared_symbols():
        stem = name[:-len("_stats")] if name.endswith("_stats") else name[:-len("_apply")] if name.endswith("_apply") else name
        assert name in doc or stem in doc, name
