"""Generate tensorboard.npz: every SummaryWriter call the reference's training_report (train.py) makes, on the CPU.

    python tests/golden/make_tensorboard_golden.py        (needs /root/reference)

training_report, utils/loss_utils.py's l1_loss and utils/image_utils.py's psnr are taken out of the reference's sources
with `ast` and executed on their own, so none of train.py's imports (the rasterizer, the scene, the games) is needed.
They run with a writer that records each call, a scene of named views whose original_image is bytes / 255 in float32 (as
PILtoTorch makes it), a renderFunc that returns a seeded image per view (values outside [0, 1] too) and a model whose
get_opacity is the sigmoid of seeded logits.

Stored per case `<c>`: the inputs (`<c>/iteration`, `<c>/test_iterations`, `<c>/loss`, `<c>/l1`, `<c>/elapsed`, per split
`<c>/<split>/names`, `/renders` [n,3,H,W] float32, `/gt` [n,H,W,3] uint8, and `<c>/opacity_logits` [P,1]) and the calls
in order: `<c>/call/<k>/method`, `/tag`, `/step` and `/value` (a float64 scalar, or the float32 array the writer got)."""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
H, W = 4, 6

# (name, n_train, n_test, iteration, test_iterations)
CASES = (
    ("outside", 12, 7, 3, [7, 10]),           # not a test iteration: the three scalars only
    ("first", 12, 7, 7, [7, 10]),             # the first listed test iteration: renders and ground truth; 12 train views wrap
    ("later", 12, 7, 10, [7, 10]),            # a later one: renders only
    ("empty_test", 4, 0, 7, [7]),             # no test views; four train views, so indices 5..25 wrap to 1, 2, 3, 0, 1
    ("few_test", 40, 3, 7, [7]),              # three test views (fewer than five); 40 train views: no wrap
    ("first_unreached", 12, 7, 7, [30, 7]),   # the first listed value is later than this one: no ground truth
)


def _functions(path, names):
    """The named top-level functions of a reference source file, compiled on their own."""
    tree = ast.parse(open(path).read(), path)
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names), path
    return ast.Module(body=body, type_ignores=[])


def reference_functions():
    ns = {"torch": torch, "Scene": object}
    for path, names in (("utils/loss_utils.py", ["l1_loss"]), ("utils/image_utils.py", ["psnr"]), ("train.py", ["training_report"])):
        exec(compile(_functions(os.path.join(REF, path), names), path, "exec"), ns)
    return ns


class Recorder:
    """SummaryWriter's add_scalar / add_images / add_histogram, recorded as (method, tag, step, value)."""

    def __init__(self):
        self.calls = []

    def add_scalar(self, tag, value, global_step=None):
        self.calls.append(("add_scalar", tag, global_step, float(value)))

    def add_images(self, tag, img, global_step=None):
        self.calls.append(("add_images", tag, global_step, np.array(img.numpy(), dtype=np.float32)))

    def add_histogram(self, tag, values, global_step=None):
        self.calls.append(("add_histogram", tag, global_step, np.array(values.numpy(), dtype=np.float32)))


class _Image:
    """original_image: `.to("cuda")` hands back the CPU tensor."""

    def __init__(self, t):
        self.t = t

    def to(self, *args, **kwargs):
        return self.t


class _View:
    def __init__(self, name, render, gt):
        self.image_name, self.render = name, render
        self.original_image = _Image(torch.from_numpy(gt).permute(2, 0, 1) / 255.0)


def case_inputs(seed, n_train, n_test):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for split, n in (("train", n_train), ("test", n_test)):
        out[f"{split}/names"] = np.array([f"{split}_{seed}_{i:03d}" for i in range(n)])
        out[f"{split}/renders"] = (torch.rand(n, 3, H, W, generator=g) * 1.4 - 0.2).numpy()
        out[f"{split}/gt"] = torch.randint(0, 256, (n, H, W, 3), generator=g, dtype=torch.uint8).numpy()
    out["opacity_logits"] = (torch.randn(50 + seed, 1, generator=g) * 3).numpy()
    out["loss"], out["l1"], out["elapsed"] = (torch.rand(3, generator=g) * torch.tensor([0.3, 0.2, 4.0])).numpy()    # float32
    return out


def run_case(ns, inp, iteration, test_iterations):
    views = {s: [_View(str(n), torch.from_numpy(r), gt) for n, r, gt in zip(inp[f"{s}/names"], inp[f"{s}/renders"], inp[f"{s}/gt"])]
             for s in ("train", "test")}
    opacity = torch.sigmoid(torch.from_numpy(inp["opacity_logits"]))
    gaussians = type("G", (), {"get_opacity": opacity, "get_xyz": torch.zeros(opacity.shape[0], 3)})()
    scene = type("S", (), {"getTrainCameras": lambda self: views["train"], "getTestCameras": lambda self: views["test"],
                           "gaussians": gaussians})()
    w = Recorder()
    Ll1 = torch.tensor(inp["l1"], dtype=torch.float32)
    loss = torch.tensor(inp["loss"], dtype=torch.float32)
    ns["training_report"](w, iteration, Ll1, loss, ns["l1_loss"], float(inp["elapsed"]), test_iterations, scene,
                          lambda view, *args: {"render": view.render}, ())
    return w.calls


def main(out=os.path.join(HERE, "tensorboard.npz")):
    ns = reference_functions()
    arrays = {}
    for seed, (name, n_train, n_test, iteration, test_iterations) in enumerate(CASES):
        inp = case_inputs(seed, n_train, n_test)
        for k, v in inp.items():
            arrays[f"{name}/{k}"] = np.asarray(v)
        arrays[f"{name}/iteration"] = np.int64(iteration)
        arrays[f"{name}/test_iterations"] = np.array(test_iterations, dtype=np.int64)
        calls = run_case(ns, inp, iteration, test_iterations)
        for k, (method, tag, step, value) in enumerate(calls):
            p = f"{name}/call/{k}/"
            arrays[p + "method"], arrays[p + "tag"], arrays[p + "step"] = np.array(method), np.array(tag), np.int64(step)
            arrays[p + "value"] = np.float64(value) if method == "add_scalar" else value
        print(f"{name}: {len(calls)} calls")
    np.savez_compressed(out, **arrays)
    print(f"wrote {out}")


if __name__ == "__main__":
    sys.exit(main())
