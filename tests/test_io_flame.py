"""CPU-only: gs_flame checkpoints against tests/golden/flame, written by the reference's own GaussianFlameModel.save_ply
(tests/golden/make_flame_golden.py): the reader returns what the reference saved, with the pickled point_cloud read without
the reference importable; the writer reproduces the reference's point_cloud.ply byte for byte and its flame_params.pt keys
and tensors."""
import os

import numpy as np
import torch

from gms_b200 import io_ply

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flame")
PLY = os.path.join(GOLD, "point_cloud.ply")


def _expected():
    return dict(np.load(os.path.join(GOLD, "expected.npz")))


def test_reader_matches_the_reference_checkpoint():
    e = _expected()
    c = io_ply.load_flame_model(PLY)
    for k in ("_xyz", "_scaling", "_rotation", "_opacity", "alpha", "_vertices_enlargement", "_flame_shape", "_flame_exp",
              "_flame_pose", "_flame_neck_pose", "_flame_trans", "_features_dc", "_features_rest"):
        np.testing.assert_array_equal(c[k].numpy(), e[k], err_msg=k)
    np.testing.assert_array_equal(c["faces"].numpy(), e["faces"])
    assert c["faces"].dtype == torch.int64 and "_scales" not in c
    pc = c["point_cloud"]       # FLAMEPointCloud of the reference's code, kept as an opaque tuple of its fields
    assert isinstance(pc, tuple) and len(pc) == 14
    np.testing.assert_array_equal(pc[4].numpy(), e["faces"])


def test_writer_reproduces_the_reference_files(tmp_path):
    e = _expected()
    c = io_ply.load_flame_model(PLY)
    out = str(tmp_path / "point_cloud.ply")
    flame = {k: torch.tensor(e[k]) for k in io_ply.FLAME_KEYS[:6]}
    io_ply.write_flame_checkpoint(out, torch.tensor(e["_xyz"]), torch.tensor(e["_features_dc"]), torch.tensor(e["_features_rest"]),
                                  torch.tensor(e["_opacity"]), torch.tensor(e["_scaling"]), torch.tensor(e["_rotation"]), flame,
                                  torch.tensor(e["faces"]), torch.tensor(e["alpha"]), point_cloud=c["point_cloud"])
    assert open(out, "rb").read() == open(PLY, "rb").read()
    ours = torch.load(out.replace("point_cloud.ply", "flame_params.pt"), weights_only=False, pickle_module=io_ply._pickle_module)
    theirs = torch.load(PLY.replace("point_cloud.ply", "flame_params.pt"), weights_only=False, pickle_module=io_ply._pickle_module)
    assert list(ours) == list(theirs) == list(io_ply.FLAME_KEYS)
    for k in io_ply.FLAME_KEYS[:-1]:
        assert type(ours[k]) is type(theirs[k]), k
        np.testing.assert_array_equal(ours[k].detach().numpy(), theirs[k].detach().numpy(), err_msg=k)
