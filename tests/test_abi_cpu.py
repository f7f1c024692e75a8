"""CPU: the C-ABI library loads and exports every declared symbol; the module mirrors the reference
surface (665-key state_dict, attributes, strict loading) and refuses to run without CUDA."""
import json
import os
import re

import pytest
import torch

from conftest import GOLDEN_DIR, ROOT


def test_library_exports_every_declared_symbol_of_abi_version_2():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "sta_b200.h")).read()
    names = sorted(set(re.findall(r"\b(sta_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert L.sta_version() == 2


def test_module_surface_matches_reference():
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    m = STA()
    spec = json.load(open(os.path.join(GOLDEN_DIR, "state_dict_spec.json")))
    sd = m.state_dict()
    assert list(sd.keys()) == [k for k, _ in spec]
    assert all(list(sd[k].shape) == s for k, s in spec)
    assert sum(p.numel() for p in m.parameters()) == 438455505  # slam.py:46
    d = "downstream_head_pts.dpt.scratch."
    assert sd[d + "layer1_rn.weight"].data_ptr() == sd[d + "layer_rn.0.weight"].data_ptr()  # aliased Parameter
    for attr, val in (("patch_size", 16), ("enc_depth", 24), ("enc_embed_dim", 1024), ("dec_depth", 12),
                      ("dec_embed_dim", 768)):
        assert getattr(m, attr) == val
    assert m.depth_mode == ("exp", -float("inf"), float("inf")) and m.conf_mode == ("exp", 1, float("inf"))
    assert m.patch_embed.patch_size == (16, 16)
    for name in ("_encode_image", "_decode_stereo", "head_pose_s", "head_pts", "forward", "load_state_dict",
                 "set_freeze"):
        assert callable(getattr(m, name))


def test_strict_load_rejects_bad_state_dicts():
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    m = STA()
    sd = dict(m.state_dict())
    sd.pop("dec_norm.weight")
    with pytest.raises(RuntimeError):
        m.load_state_dict(sd, strict=True)
    sd = dict(m.state_dict())
    sd["extra.weight"] = torch.zeros(1)
    with pytest.raises(RuntimeError):
        m.load_state_dict(sd, strict=True)
    m.load_state_dict(dict(m.state_dict()), strict=True)


def test_non_default_configuration_is_refused():
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    with pytest.raises(NotImplementedError):
        STA(enc_depth=12)
    with pytest.raises(NotImplementedError):
        STA(head_type="linear")


def test_no_cpu_fallback():
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    m = STA()
    with pytest.raises(RuntimeError, match="CUDA"):
        m._encode_image(torch.zeros(1, 3, 32, 32), torch.tensor([[32, 32]]), normalize=False)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.head_pose_s(torch.zeros(1, 768))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "vista_slam_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                # no import of, and no path into, the oracle package; the word may only appear in comments that point at
                # oracle/<file> as the checker of a kernel
                assert "import oracle" not in src and "from oracle" not in src, (dp, f)
                assert "oracle" not in src.replace("oracle/", "").lower(), (dp, f)


def test_library_built_with_other_nvcc_flags_is_stale(tmp_path, monkeypatch):
    """A library whose recorded nvcc flags differ from the current ones (e.g. another GPU architecture) is rebuilt,
    however new it is."""
    from vista_slam_b200 import build as b
    lib = tmp_path / "libsta_b200.so"
    lib.write_bytes(b"")
    stamp = tmp_path / "nvcc_flags.txt"
    monkeypatch.setattr(b, "LIB", str(lib))
    monkeypatch.setattr(b, "STAMP", str(stamp))
    monkeypatch.setattr(b, "CSRC", str(tmp_path))  # no sources here: only the flags decide
    assert b._stale()  # no record of the flags
    stamp.write_text(" ".join(b.NVCC_FLAGS))
    assert not b._stale()
    stamp.write_text(" ".join(b.NVCC_FLAGS).replace("sm_90a", "sm_100a"))
    assert b._stale()
