"""Hires-fix upscalers, host side: Pillow's resampling tables and paste arithmetic against PIL itself (bitwise), sdwui's
tile geometry, the RRDBNet key layouts, and how LocalGPUWorker routes `hr_upscaler` (engine double)."""
import types

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import upscale_oracle as UO

SIZES = [(512, 1024), (1024, 512), (2048, 1024), (97, 311), (311, 97), (100, 29), (29, 100), (513, 127), (127, 513),
         (64, 17), (17, 64), (768, 1000), (1000, 768), (5, 3), (3, 5), (1, 7), (7, 1), (250, 251), (251, 250), (600, 173),
         (333, 100), (1024, 1023)]


def _rgb(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _apply(img, filt, w, h):
    """the kernels' arithmetic in numpy: Pillow's horizontal pass, then the vertical one, each skipped if unchanged"""
    from b200sd import upscale as U
    x = img.astype(np.int64)
    for axis, n_out in ((1, w), (0, h)):
        n_in = x.shape[axis]
        if n_in == n_out:
            continue
        bounds, kk = U.pil_tables(filt, n_in, n_out)
        xm = np.moveaxis(x, axis, 0)
        out = np.zeros((n_out,) + xm.shape[1:], np.int64)
        for o in range(n_out):
            first, count = bounds[o]
            s = np.full(xm.shape[1:], 1 << (U.PRECISION_BITS - 1), np.int64)
            for t in range(count):
                s += xm[first + t] * int(kk[o, t])
            out[o] = np.clip(s >> U.PRECISION_BITS, 0, 255)
        x = np.moveaxis(out, 0, axis)
    return x.astype(np.uint8)


@pytest.mark.parametrize("filt", ["lanczos", "nearest"])
def test_pillow_tables_equal_pil_resize(filt):
    pil_filter = Image.LANCZOS if filt == "lanczos" else Image.NEAREST
    for i, (a, b) in enumerate(SIZES):
        img = _rgb(i, 23 + i % 5, a)                     # horizontal a -> b
        want = np.array(Image.fromarray(img).resize((b, img.shape[0]), pil_filter))
        assert np.array_equal(_apply(img, filt, b, img.shape[0]), want), (filt, a, b)
        img = _rgb(100 + i, a, 19)                        # vertical a -> b
        want = np.array(Image.fromarray(img).resize((19, b), pil_filter))
        assert np.array_equal(_apply(img, filt, 19, b), want), (filt, a, b)
    img = _rgb(7, 131, 257)                               # both axes, ratio under 1/3 on one of them
    for w, h in ((512, 40), (37, 300), (256, 256)):
        want = np.array(Image.fromarray(img).resize((w, h), pil_filter))
        assert np.array_equal(_apply(img, filt, w, h), want), (filt, w, h)


def _combine_np(tiles, ys, xs, h, w, overlap):
    """the combine kernel's arithmetic in numpy (paste order per output pixel, Pillow's DIV255 blend)"""
    from b200sd import upscale as U
    mask = U.blend_mask(max(overlap, 1)).astype(np.int64)
    th, tw = tiles.shape[2], tiles.shape[3]
    out = np.zeros((h, w, 3), np.int64)

    def blend(a, under, over):
        t = under * (255 - a) + over * a + 128
        return ((t >> 8) + t) >> 8

    for r, y in enumerate(ys):
        row = np.zeros((th, w, 3), np.int64)
        for c, x in enumerate(xs):
            t = tiles[r, c].astype(np.int64)
            for xx in range(max(0, -x), min(tw, w - x)):
                X = x + xx
                row[:, X] = blend(mask[xx], row[:, X], t[:, xx]) if (x != 0 and xx < overlap) else t[:, xx]
        for yy in range(max(0, -y), min(th, h - y)):
            Y = y + yy
            out[Y] = blend(mask[yy], out[Y], row[yy]) if (y != 0 and yy < overlap) else row[yy]
    return out.astype(np.uint8)


@pytest.mark.parametrize("w,h,tile,overlap", [(160, 120, 48, 8), (100, 60, 48, 4), (30, 20, 48, 8), (97, 53, 32, 6)])
def test_muldiv255_blend_equals_combine_grid(w, h, tile, overlap):
    from b200sd import upscale as U
    ys, xs = U.split_grid(w, h, tile, tile, overlap)
    rng = np.random.default_rng(w * h)
    tiles = rng.integers(0, 256, (len(ys), len(xs), tile, tile, 3), dtype=np.uint8)
    grid = UO.Grid([[y, tile, [[x, tile, Image.fromarray(tiles[r, c])] for c, x in enumerate(xs)]] for r, y in enumerate(ys)],
                   tile, tile, w, h, overlap)
    assert np.array_equal(_combine_np(tiles, ys, xs, h, w, overlap), np.array(UO.combine_grid(grid)))


@pytest.mark.parametrize("w,h", [(512, 512), (1024, 1024), (513, 700), (200, 191), (100, 60), (192, 192), (193, 400)])
def test_tile_geometry_equals_split_grid(w, h):
    from b200sd import upscale as U
    img = Image.fromarray(_rgb(w, h, w))
    grid = UO.split_grid(img, 192, 192, 8)
    ys, xs = U.split_grid(w, h, 192, 192, 8)
    assert ys == [y for y, _, _ in grid.tiles] and xs == [x for x, _, _ in grid.tiles[0][2]]
    tiles = U.crop_tiles(torch.from_numpy(np.array(img))[None], ys, xs, 192, 192).numpy()
    want = np.stack([np.array(t) for _, _, row in grid.tiles for _, _, t in row])
    assert np.array_equal(tiles, want)


def _old_layout(sd):
    """basicsr keys -> old ESRGAN keys"""
    nb = len({int(k.split(".")[1]) for k in sd if k.startswith("body.")})
    ren = {"conv_first": "model.0", "conv_up1": "model.3", "conv_up2": "model.6", "conv_hr": "model.8",
           "conv_last": "model.10", "conv_body": f"model.1.sub.{nb}"}
    out = {}
    for k, v in sd.items():
        stem, _, leaf = k.rpartition(".")
        if stem in ren:
            out[f"{ren[stem]}.{leaf}"] = v
        else:
            _, i, rdb, conv = stem.split(".")
            out[f"model.1.sub.{i}.RDB{rdb[3:]}.{conv}.0.{leaf}"] = v
    return out


@pytest.mark.parametrize("nb", [1, 3])
def test_both_key_layouts_load_into_the_oracle(nb, tmp_path, monkeypatch):
    from b200sd import upscale as U
    sd = U.synthetic_state_dict(nb, seed=nb)
    torch.save({"params_ema": sd}, tmp_path / "new.pth")
    torch.save(_old_layout(sd), tmp_path / "old.pth")
    monkeypatch.setenv("B200SD_UPSCALER_DIR", str(tmp_path))
    a, b = U.load_state_dict("new"), U.load_state_dict("old")
    assert U.num_blocks(a) == U.num_blocks(b) == nb and set(a) == set(b)
    x = torch.rand((1, 3, 12, 10), generator=torch.Generator().manual_seed(0))
    ya, yb = UO.rrdbnet(a, x), UO.rrdbnet(b, x)
    assert ya.shape == (1, 3, 48, 40) and torch.equal(ya, yb)
    torch.save({"conv.weight": torch.zeros(1)}, tmp_path / "other.pth")
    with pytest.raises(U.UnsupportedUpscaler):
        U.load_state_dict("other")
    with pytest.raises(U.UnsupportedUpscaler):
        U.load_state_dict("missing")


class _NotAStateDict:
    pass


def test_unreadable_model_files_are_unsupported_upscalers(tmp_path, monkeypatch):
    """files torch.load(weights_only=True) refuses, that do not hold a dict, or that are no checkpoint at all are refused
    as UnsupportedUpscaler, which the worker turns into its "Latent" fallback"""
    from b200sd import upscale as U
    monkeypatch.setenv("B200SD_UPSCALER_DIR", str(tmp_path))
    torch.save({"conv_first.weight": _NotAStateDict()}, tmp_path / "pickled.pth")
    torch.save([torch.zeros(1)], tmp_path / "alist.pth")
    (tmp_path / "garbage.pth").write_bytes(b"not a checkpoint")
    (tmp_path / "garbage.safetensors").write_bytes(b"\x00" * 16)
    torch.save({"body.x.rdb1.conv1.weight": torch.zeros(1)}, tmp_path / "badkeys.pth")
    for stem in ("pickled", "alist", "garbage", "badkeys"):
        with pytest.raises(U.UnsupportedUpscaler):
            U.load_state_dict(stem)
    (tmp_path / "garbage.pth").unlink()
    with pytest.raises(U.UnsupportedUpscaler):
        U.load_state_dict("garbage")   # the .safetensors twin


def test_synthetic_rrdbnet_activations_stay_order_one():
    from b200sd import upscale as U
    y = UO.rrdbnet(U.synthetic_state_dict(23, seed=1), torch.rand((1, 3, 16, 16), generator=torch.Generator().manual_seed(1)))
    assert torch.isfinite(y).all() and 1e-3 < float(y.std()) < 10.0


def test_latent_tables_match_interpolate_on_cpu():
    """the tables applied in fp64 reproduce F.interpolate to fp32 rounding (nearest modes exactly)"""
    from b200sd import upscale as U
    x = torch.randn((2, 4, 13, 9), generator=torch.Generator().manual_seed(0))
    for name, (mode, aa) in U.LATENT_MODES.items():
        if name == "Latent":
            continue
        for ho, wo in ((26, 18), (40, 21), (13, 9), (7, 5)):
            want = torch.nn.functional.interpolate(x, size=(ho, wo), mode=mode, antialias=aa)
            (ix, wx), (iy, wy) = [(torch.from_numpy(i).long(), torch.from_numpy(w).double())
                                  for i, w in (U._latent_axis(mode, aa, 9, wo), U._latent_axis(mode, aa, 13, ho))]
            rows = (x.double()[:, :, :, ix] * wx).sum(-1)           # [b, c, 13, wo]
            got = (rows[:, :, iy, :] * wy[..., None]).sum(3)         # [b, c, ho, wo]
            if mode.startswith("nearest"):
                assert torch.equal(got.float(), want), (name, ho, wo)
            else:
                assert torch.allclose(got.float(), want, atol=2e-6, rtol=1e-5), (name, ho, wo, float((got - want).abs().max()))


# ------------------------------------------------------------------------------------------------ worker routing
class _Engine:
    def __init__(self):
        self.interrupted = False
        self.variation = (None, 0.0)
        self.device = torch.device("cpu")
        self.clip_cfg = types.SimpleNamespace(vocab=1000)
        self.unet_cfg = types.SimpleNamespace(adm_in_channels=0)
        self.calls = []

    def txt2img_hires(self, tok, neg, seed, **kw):
        self.calls.append(kw)
        b = tok.shape[0]
        s = kw["hr_scale"]
        return torch.zeros((b, int(kw["height"] * s), int(kw["width"] * s), 3), dtype=torch.uint8)


@pytest.fixture()
def worker(monkeypatch):
    from b200sd import upscale
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker
    monkeypatch.delenv("B200SD_UPSCALER_DIR", raising=False)
    monkeypatch.setattr(upscale, "model", lambda stem, device: None)   # packing is covered above; routing only here
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    eng = _Engine()
    return LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0), eng


def _payload(**kw):
    p = {"prompt": "a b", "negative_prompt": "", "seed": 30, "subseed": 4, "subseed_strength": 0, "batch_size": 2,
         "n_iter": 1, "steps": 4, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0,
         "enable_hr": True, "hr_scale": 2.0, "denoising_strength": 0.6}
    p.update(kw)
    return p


SERVED = ["Latent (antialiased)", "Latent (bicubic)", "Latent (bicubic antialiased)", "Latent (nearest)",
          "Latent (nearest-exact)", "None", "Lanczos", "Nearest", "R-ESRGAN 4x+", "R-ESRGAN 4x+ Anime6B", "ESRGAN_4x",
          "4x-UltraSharp"]


@pytest.mark.parametrize("name", SERVED)
def test_served_upscalers_reach_the_engine(worker, name):
    wk, eng = worker
    wk.request(_payload(hr_upscaler=name, override_settings={"ESRGAN_tile": 128, "ESRGAN_tile_overlap": 16}), None, False)
    kw = eng.calls[-1]
    assert kw["upscaler"] == name and wk.response["tensors"].shape == (2, 128, 128, 3)
    esrgan = name in ("R-ESRGAN 4x+", "R-ESRGAN 4x+ Anime6B", "ESRGAN_4x", "4x-UltraSharp")
    assert (kw.get("upscaler_tile"), kw.get("upscaler_overlap")) == ((128, 16) if esrgan else (None, None))


@pytest.mark.parametrize("name", ["R-ESRGAN 2x+", "R-ESRGAN General 4xV3", "R-ESRGAN General WDN 4xV3",
                                  "R-ESRGAN AnimeVideo", "SwinIR 4x", "ScuNET GAN", "LDSR", "DAT x4"])
def test_unserved_upscalers_warn_and_use_latent(worker, name, monkeypatch):
    from scripts.spartan import local_worker
    wk, eng = worker
    warned = []
    monkeypatch.setattr(local_worker.logger, "warning", lambda msg, *a, **k: warned.append(msg))
    wk.request(_payload(hr_upscaler=name), None, False)
    assert "upscaler" not in eng.calls[-1] and any(name in m for m in warned)


def test_a_file_that_is_not_a_4x_rrdbnet_falls_back(worker, tmp_path, monkeypatch):
    from b200sd import upscale
    wk, eng = worker
    monkeypatch.setattr(upscale, "model", lambda stem, device: upscale.load_state_dict(stem))
    monkeypatch.setenv("B200SD_UPSCALER_DIR", str(tmp_path))
    torch.save({"conv.weight": torch.zeros(1)}, tmp_path / "srvgg.pth")
    wk.request(_payload(hr_upscaler="srvgg"), None, False)
    assert "upscaler" not in eng.calls[-1]


@pytest.mark.parametrize("extra", [{}, {"hr_upscaler": "Latent"}, {"hr_upscaler": None}])
def test_latent_payloads_reach_the_engine_with_todays_arguments(worker, extra):
    wk, eng = worker
    wk.request(_payload(**extra), None, False)
    assert set(eng.calls[-1]) == {"steps", "cfg_scale", "height", "width", "hr_scale", "hr_steps", "denoising_strength",
                                  "sampler", "scheduler"}


def test_controlnet_with_hires_is_still_refused(worker):
    from scripts.spartan.worker import InvalidWorkerResponse
    wk, eng = worker
    unit = {"enabled": True, "module": "none", "model": "control_canny", "weight": 1.0,
            "image": np.zeros((64, 64, 3), np.uint8)}
    with pytest.raises(InvalidWorkerResponse):
        wk.request(_payload(hr_upscaler="Lanczos", alwayson_scripts={"controlnet": {"args": [unit]}}), None, False)
    assert not eng.calls
