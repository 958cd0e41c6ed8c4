"""CPU-only: the LPIPS float64 restatement (tests/lpips_oracle.py) against torchvision's VGG16 structure and the reference's
own LPIPS head (lpips.npz); loading the weight files (keys, shapes, the cache directory, and that nothing is fetched); and
the JSON and printed lines of cli.metrics --lpips with a stub scorer."""
import io
import json
import os
import socket
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import lpips_oracle
from gms_b200 import _lib, lpips
from gms_b200.cli import metrics as cli_metrics


def test_oracle_layers_are_torchvision_vgg16_features():
    tv = pytest.importorskip("torchvision")
    feats = tv.models.vgg16(weights=None).features            # structure only: no weights, nothing downloaded
    assert len(lpips_oracle.LAYERS) == 30 and len(feats) == 31
    for i, (layer, mod) in enumerate(zip(lpips_oracle.LAYERS, feats)):
        if layer[0] == "conv":
            assert isinstance(mod, torch.nn.Conv2d) and layer[1] == i, i
            assert (mod.in_channels, mod.out_channels) == layer[2:] and mod.kernel_size == (3, 3), i
            assert mod.padding == (1, 1) and mod.stride == (1, 1) and mod.bias is not None, i
        elif layer[0] == "relu":
            assert isinstance(mod, torch.nn.ReLU), i
        else:
            assert isinstance(mod, torch.nn.MaxPool2d) and mod.kernel_size == 2 and mod.stride == 2 and not mod.ceil_mode, i
    chans = [lpips_oracle.LAYERS[t - 2][3] for t in lpips_oracle.TARGET_LAYERS]    # the conv before each target ReLU
    assert chans == list(lpips.LIN_CHANNELS) == list(lpips_oracle.LIN_CHANNELS)
    assert [layer[1] for layer in lpips_oracle.LAYERS if layer[0] == "conv"] == list(lpips.CONV_INDEX)


def test_oracle_head_reproduces_the_reference(golden_dir):
    d = np.load(os.path.join(golden_dir, "lpips.npz"))
    for c in range(int(d["n_cases"])):
        fx = [torch.from_numpy(d[f"case{c}_x{l}"]).double() for l in range(5)]
        fy = [torch.from_numpy(d[f"case{c}_y{l}"]).double() for l in range(5)]
        lin = {f"lin{l}.model.1.weight": torch.from_numpy(d[f"case{c}_lin{l}"]) for l in range(5)}
        got = float(lpips_oracle.head(fx, fy, lin)[5])
        ref = float(d[f"case{c}_lpips"].reshape(()))
        assert abs(got - ref) <= 1e-6 * abs(ref), (c, got, ref)          # the reference computes in float32
        if c == 2:
            assert got == ref == 0.0


def test_packed_layout_and_loading_from_both_file_formats(tmp_path):
    vp, lp, vgg16, lin = lpips_oracle.write_weight_files(tmp_path, seed=1)
    packed = lpips.pack_weights(torch.load(vp, weights_only=True), torch.load(lp, weights_only=True))
    assert packed.numel() == _lib.LPIPS_WEIGHT_FLOATS
    # conv1_1: [64][32], K ordered (ky, kx, ci) and padded with zeros; then its bias; conv1_2 follows
    w0 = packed[:64 * 32].view(64, 32)
    assert torch.equal(w0[:, :27], vgg16["features.0.weight"].permute(0, 2, 3, 1).reshape(64, 27))
    assert torch.equal(w0[:, 27:], torch.zeros(64, 5))
    assert torch.equal(packed[64 * 32:64 * 33], vgg16["features.0.bias"])
    assert torch.equal(packed[64 * 33:64 * 33 + 64 * 576].view(64, 576), vgg16["features.2.weight"].permute(0, 2, 3, 1).reshape(64, 576))
    assert torch.equal(packed[-1472:], torch.cat([lin[f"lin{l}.model.1.weight"].flatten() for l in range(5)]))


def test_key_and_shape_errors_name_the_key(tmp_path):
    vgg16, lin = lpips_oracle.seeded_state_dicts(2)
    bad = dict(vgg16)
    del bad["features.12.bias"]
    with pytest.raises(KeyError, match=r"features\.12\.bias"):
        lpips.pack_weights(bad, lin)
    bad = dict(vgg16)
    bad["features.26.weight"] = torch.zeros(512, 512, 1, 1)
    with pytest.raises(ValueError, match=r"features\.26\.weight.*\(512, 512, 3, 3\)"):
        lpips.pack_weights(bad, lin)
    bad = dict(lin)
    del bad["lin3.model.1.weight"]
    with pytest.raises(KeyError, match=r"lin3\.model\.1\.weight"):
        lpips.pack_weights(vgg16, bad)
    # classifier.* is never read, whatever it holds
    other = dict(vgg16)
    other["classifier.6.weight"] = "not a tensor"
    assert torch.equal(lpips.pack_weights(other, lin), lpips.pack_weights(vgg16, lin))


def test_cache_dir_follows_torch_home(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(torch.hub, "_hub_dir", None)
    assert lpips.cache_dir() == os.path.join(str(tmp_path / "th"), "hub", "checkpoints")
    os.makedirs(lpips.cache_dir())
    lpips_oracle.write_weight_files(lpips.cache_dir(), seed=0)
    seen = []
    monkeypatch.setattr(lpips, "pack_weights", lambda v, l, vp, lp: seen.append((vp, lp)) or torch.zeros(1))
    with pytest.raises(ValueError):            # the zero-length stand-in is refused by Lpips itself, after loading
        lpips.Lpips.from_cache()
    assert seen == [(os.path.join(lpips.cache_dir(), "vgg16-397923af.pth"), os.path.join(lpips.cache_dir(), "vgg.pth"))]


def test_missing_file_is_named_and_nothing_is_fetched(tmp_path, monkeypatch):
    def no_network(*a, **k):
        raise AssertionError("network access attempted")
    monkeypatch.setattr(socket, "socket", no_network)
    monkeypatch.setattr(socket, "create_connection", no_network)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_network)
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_network)
    vp, lp = str(tmp_path / "vgg16-397923af.pth"), str(tmp_path / "vgg.pth")
    for present in ((), ("vgg",), ("vgg16",)):
        for f in (vp, lp):
            if os.path.exists(f):
                os.remove(f)
        if present:
            torch.save({}, lp if present == ("vgg",) else vp)
        with pytest.raises(FileNotFoundError) as e:
            lpips.Lpips.from_cache(str(tmp_path))
        msg = str(e.value)
        assert vp in msg and lp in msg and "does not download" in msg, msg


def _method_tree(tmp_path, names):
    model = tmp_path / "model"
    for m in ("ours_30", "ours_7"):
        for sub in ("renders_gs_flat", "gt"):
            os.makedirs(model / "test" / m / sub)
        for n in names:
            (model / "test" / m / "renders_gs_flat" / n).write_bytes(b"")
    return model


def test_metrics_cli_lpips_json_and_printed_lines(tmp_path):
    model = _method_tree(tmp_path, ("00002.png", "00000.png", "00001.png"))
    rng = np.random.default_rng(1)
    values = {}
    scorer = object()

    def fake_score(renders_dir, gt_dir, device, lp):
        assert lp is scorer
        names = os.listdir(renders_dir)
        pv = torch.tensor(rng.uniform(0.5, 40.0, (len(names), 4)), dtype=torch.float64)
        lv = torch.tensor(rng.uniform(0.0, 0.5, len(names)), dtype=torch.float32)
        values[renders_dir.parent.name] = (names, pv, lv)
        return names, pv, lv

    buf = io.StringIO()
    with redirect_stdout(buf):
        cli_metrics.evaluate("gs_flat", [str(model)], score=fake_score, lpips=scorer)
    results = json.loads((model / "results_gs_flat.json").read_text())
    per_view = json.loads((model / "per_view_gs_flat.json").read_text())
    lines = buf.getvalue().split("\n")
    for m, (names, pv, lv) in values.items():
        assert list(results[m]) == ["SSIM", "PSNR", "LPIPS"] and list(per_view[m]) == ["SSIM", "PSNR", "LPIPS"]
        assert list(per_view[m]["LPIPS"]) == names
        assert list(per_view[m]["LPIPS"].values()) == lv.tolist()
        assert results[m]["LPIPS"] == lv.mean().item()
        i = lines.index(f"Method: {m}")
        assert lines[i + 1:i + 5] == ["  SSIM : {:>12.7f}".format(pv[:, 1].float().mean()),
                                      "  PSNR : {:>12.7f}".format(pv[:, 2].float().mean()),
                                      "  LPIPS: {:>12.7f}".format(lv.mean()), ""]
