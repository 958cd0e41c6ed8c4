"""CPU-only: metrics.npz (the reference's own l1_loss / ssim / psnr, tests/golden/make_metrics_golden.py) agrees with the
float64 restatement of the four view metrics that the GPU tests also compare gms_image_metrics with."""
import math
import os

import numpy as np
import pytest
import torch

from metrics_restated import metrics64

PROTOCOLS = ("training_report", "metrics")


@pytest.mark.parametrize("protocol", PROTOCOLS)
def test_fixture_matches_the_float64_restatement(golden_dir, protocol):
    d = np.load(os.path.join(golden_dir, "metrics.npz"))
    for i in range(int(d["n_cases"])):
        ref = d[f"case{i}_{protocol}"]
        got = metrics64(torch.from_numpy(d[f"case{i}_img"]), torch.from_numpy(d[f"case{i}_gt"]), protocol)
        # the reference computes in float32: L1 / SSIM to ~1e-7, PSNR to ~1e-5 dB
        assert abs(got[0] - ref[0]) <= 2e-6 and abs(got[1] - ref[1]) <= 2e-6, (i, got, ref)
        for k in (2, 3):
            if math.isinf(ref[k]):
                assert math.isinf(got[k]) and got[k] > 0, (i, k)
            else:
                assert abs(got[k] - ref[k]) <= 1e-4, (i, k, got[k], ref[k])


def test_per_channel_psnr_differs_from_the_global_one(golden_dir):
    """training_report averages one PSNR per channel (psnr() on [C,H,W] views it as C rows): not the PSNR of the whole image."""
    d = np.load(os.path.join(golden_dir, "metrics.npz"))
    r = d["case0_training_report"]
    assert abs(r[3] - r[2]) > 1e-4
