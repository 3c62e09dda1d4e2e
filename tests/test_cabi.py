"""CPU-side checks of the C-ABI boundary: the library builds/loads and exports every symbol
declared in include/lion_b200.h (no compute calls without a GPU)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "lion_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lion_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from lion_b200 import _lib
    lib = _lib.lib()
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), "liblion_b200.so does not export %s" % n
    assert set(names) == set(_lib.EXPORTS), (set(names) ^ set(_lib.EXPORTS))
    assert lib.lion_version() >= 100


def test_no_cpu_fallback():
    """The product path must fail loudly without CUDA tensors -- never fall back."""
    import torch
    from lion_b200 import _lib
    from lion_b200.third_party.pvcnn import functional as F
    with pytest.raises(_lib.LionError):
        F.ball_query(torch.zeros(1, 3, 4), torch.zeros(1, 3, 8), 0.1, 4)


def test_product_path_does_not_import_oracle():
    bad = []
    for dp, _, fs in os.walk(os.path.join(ROOT, "lion_b200")):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                s = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b|from\s+\.+oracle", s, flags=re.M):
                    bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_state_dict_key_contract():
    """Module trees expose exactly the reference's parameter names and shapes (SURVEY.md App. E;
    tests/golden/keys.json was dumped from the reference modules)."""
    import json
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    from lion_b200.models.score_sde.resnet import PriorSEDrop, PriorSEClip
    from lion_b200.models.vae_adain import Model
    keys = json.load(open(os.path.join(ROOT, "tests", "golden", "keys.json")))
    shp = lambda m: {k: list(v.shape) for k, v in m.state_dict().items()}
    cfg, cc = default_prior_cfg(), default_prior_cfg(clip=True)
    assert shp(PVCNN2Prior(cfg.sde, 1, cfg)) == keys["prior"]
    assert shp(PVCNN2Prior(cc.sde, 1, cc)) == keys["prior_clip"]
    assert shp(PriorSEDrop(cfg.sde, 128, cfg)) == keys["global"]
    assert shp(PriorSEClip(cc.sde, 128, cc)) == keys["global_clip"]
    vae = shp(Model(cfg))                     # the VAE now carries both encoders as well (SURVEY.md 8f-3)
    assert {k: v for k, v in vae.items() if k.startswith("decoder.")} == keys["vae_decoder"]
    ekeys = json.load(open(os.path.join(ROOT, "tests", "golden", "keys_encoder.json")))
    assert {k[len("style_encoder."):]: v for k, v in vae.items() if k.startswith("style_encoder.")} == ekeys["style_encoder"]
    assert {k[len("encoder."):]: v for k, v in vae.items() if k.startswith("encoder.")} == ekeys["point_encoder"]


def _header_prototypes():
    """{name: number of parameters} parsed from include/lion_b200.h"""
    src = open(os.path.join(ROOT, "include", "lion_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(lion_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        args = m.group(2).strip()
        out[m.group(1)] = 0 if args in ("", "void") else len([a for a in args.split(",") if a.strip()])
    return out


def test_ctypes_prototypes_match_the_header():
    """The host side binds every entry point with an explicit ctypes prototype (lion_b200/_lib.py);
    its arity must be the header's -- a drifted argument list would corrupt the call silently."""
    from lion_b200 import _lib
    lib = _lib.lib()
    protos = _header_prototypes()
    assert set(protos) == set(_lib.EXPORTS)
    for name, n in protos.items():
        fn = getattr(lib, name)
        assert fn.argtypes is not None and len(fn.argtypes) == n, "%s: header has %d parameters, ctypes prototype %s" % (
            name, n, None if fn.argtypes is None else len(fn.argtypes))


def test_integration_shim_names_exist():
    """Every lion_* symbol the reference-side binding in INTEGRATION.md calls is exported."""
    from lion_b200 import _lib
    lib = _lib.lib()
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    used = sorted(set(re.findall(r"_lib\.(lion_[a-z0-9_]+)", text)))
    assert len(used) >= 7
    for n in used:
        assert hasattr(lib, n), n


def test_vae_state_dict_loads_strict():
    """A reference `vae_state_dict` (style_encoder + encoder + decoder) loads with strict=True: the key contract of
    keys.json (decoder) and keys_encoder.json (both encoders, dumped from the reference's own modules)."""
    import json
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.vae_adain import Model
    from tests.synth import synth_state_dict
    G = os.path.join(ROOT, "tests", "golden")
    keys = json.load(open(os.path.join(G, "keys.json")))
    ekeys = json.load(open(os.path.join(G, "keys_encoder.json")))
    sd = {}
    for pre, shapes, seed in (("style_encoder.", ekeys["style_encoder"], 21), ("encoder.", ekeys["point_encoder"], 22),
                              ("decoder.", keys["decoder"], 13)):
        sd.update({pre + k: v for k, v in synth_state_dict(shapes, seed).items()})
    vae = Model(default_prior_cfg())
    vae.load_state_dict(sd, strict=True)
    assert set(vae.state_dict()) == set(sd)


def test_shipped_library_contains_hopper_tensor_and_bulk_copy_sass():
    """The built liblion_b200.so must carry the sm_90a-native instructions the design rests on -- wgmma (HGMMA),
    cp.async.bulk (UBLKCP), mbarriers (SYNCS) -- so that a build whose convolutions all fall back to the SIMT kernel
    (which only serves output widths that are not a multiple of 32) cannot ship.  cuobjdump needs no GPU."""
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    so = os.path.join(ROOT, "lion_b200", "csrc", "liblion_b200.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, timeout=300).stdout
    assert "sm_90a" in sass
    for op, least in (("HGMMA", 100), ("UBLKCP", 10), ("SYNCS", 50)):
        n = len(re.findall(r"\b%s\b" % op, sass))
        assert n >= least, "%s appears %d times in the SASS (expected >= %d)" % (op, n, least)
