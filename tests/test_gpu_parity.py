"""-m gpu: the CUDA path (through diff_gaussian_rasterization -> C ABI -> sm_90a kernels) against the CPU oracle.
Bit-exact for radii / tiles_touched / sort keys / point list / tile ranges / n_contrib; <= 1e-5 abs per pixel for
colour, inverse depth and final transmittance (north_star tolerance); gradients <= 2e-4 of max|ref| (float atomics
change the summation order; the oracle accumulates in double)."""
import numpy as np
import pytest
import torch

from gms_b200 import _lib, scenes
from helpers import settings_from_camera, random_gaussians
from gpu_helpers import run_gpu, run_oracle, assert_forward_parity, assert_grad_parity

pytestmark = pytest.mark.gpu


def _case(P, W, H, seed, extent=1.2, scale_mu=-2.6, **skw):
    cam = scenes.look_at_camera((2.8, 0.6, 1.1), (0, 0, 0), W, H)
    S = settings_from_camera(cam, bg=(0.1, 0.4, 0.8), **skw)
    return S, random_gaussians(P, seed=seed, extent=extent, scale_mu=scale_mu)


def _grads_in(H, W, seed):
    rs = np.random.RandomState(seed)
    return rs.randn(3, H, W).astype(np.float32), rs.randn(H, W).astype(np.float32)


@pytest.mark.parametrize("P,W,H", [(3000, 320, 208), (20000, 400, 300), (500, 64, 48), (1, 32, 32)])
def test_forward_backward_parity_random_gaussians(P, W, H):
    S, g = _case(P, W, H, seed=P)
    dC, dI = _grads_in(H, W, 1)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


def test_ragged_image_size_not_multiple_of_16():
    S, g = _case(4000, 333, 201, seed=11)
    dC, dI = _grads_in(201, 333, 2)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


@pytest.mark.parametrize("aa", [False, True])
def test_antialiasing_and_scale_modifier(aa):
    S, g = _case(3000, 256, 256, seed=5, antialiasing=aa, scale_modifier=1.3)
    dC, dI = _grads_in(256, 256, 3)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_sh_degrees(deg):
    S, g = _case(2000, 192, 160, seed=6, sh_degree=deg)
    dC, dI = _grads_in(160, 192, 4)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


def test_precomputed_colors_and_covariance():
    S, g = _case(2500, 256, 192, seed=7)
    from oracle import torch_dense
    R = torch_dense.quat_to_R(g["rotations"].double()); Mx = R * g["scales"].double()[:, None, :]
    Sg = Mx @ Mx.transpose(1, 2)
    cov = torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1).float()
    g2 = dict(means3D=g["means3D"], opacities=g["opacities"], colors_precomp=torch.rand(2500, 3), cov3D_precomp=cov)
    dC, dI = _grads_in(192, 256, 5)
    color, radii, invd, state, grads = run_gpu(S, g2, dC, dI)
    st, gref = run_oracle(S, g2, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


def test_saturating_scene_early_termination_and_long_lists():
    """Large opaque splats: tiles hold thousands of splats, T hits 1e-4, batches > 1 are exercised."""
    S, g = _case(30000, 256, 256, seed=8, extent=0.9, scale_mu=-1.6)
    dC, dI = _grads_in(256, 256, 6)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert (st.ranges[:, 1] - st.ranges[:, 0]).max() > 1000 and (st.final_T < 2e-4).mean() > 0.2
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, tol=5e-4)


def test_flat_mesh_gaussians_edge_on_slivers():
    """Mesh Gaussians (s0 ~ 2e-8) seen at grazing angles: ill-conditioned conics; canonical op order must hold."""
    p = scenes.init_mesh_gaussians(*scenes.icosphere(4), K=3, seed=2)
    from oracle import expansion as oexp
    xyz, sl, rr, _, _ = oexp.expand(p.vertices, p.faces, p._alpha, p._scale)
    sc, rot, op, feats = oexp.activate(sl, rr, p._opacity, p._features_dc, p._features_rest)
    g = dict(means3D=xyz, opacities=op, shs=feats.contiguous(), scales=sc, rotations=rot)
    cam = scenes.look_at_camera((2.2, 0.3, 0.4), (0, 0, 0), 400, 400)
    S = settings_from_camera(cam, bg=(1, 1, 1))
    dC, dI = _grads_in(400, 400, 7)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, tol=5e-4)


@pytest.mark.parametrize("fwd,bwd,tile_order,minb", [(2, 5, 1, 6), (2, 5, 0, 4), (2, 5, 1, 8), (2, 3, 1, 6), (3, 3, 0, 6), (3, 5, 1, 6)])
@pytest.mark.parametrize("with_depth", [True, False])
def test_composite_kernel_variants_agree_and_match_oracle(fwd, bwd, tile_order, minb, with_depth):
    """Forward: scalar (2, writes the per-quad survivor lists) / float2 pairs (3).  Backward: survivor-list driven (5,
    default) / predecessor that re-derives the survivors (3; also what runs after a forward without lists, e.g. fwd=3).
    Both DEPTH template variants, every launch-bounds variant, with and without the longest-first tile order."""
    S, g = _case(12000, 352, 272, seed=21, extent=1.0, scale_mu=-2.2)
    dC, dI = _grads_in(272, 352, 9)
    olds = [_lib.set_option(k, v) for k, v in (("composite_fwd", fwd), ("composite_bwd", bwd), ("tile_order", tile_order), ("bwd_minblocks", minb))]
    try:
        color, radii, invd, state, grads = run_gpu(S, g, dC, dI if with_depth else None)
    finally:
        for k, v in zip(("composite_fwd", "composite_bwd", "tile_order", "bwd_minblocks"), olds):
            _lib.set_option(k, v)
    st, gref = run_oracle(S, g, dC, dI if with_depth else None)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


@pytest.mark.parametrize("P,W,H,scale_mu", [(20000, 400, 300, -2.6), (3000, 333, 201, -2.6), (600, 640, 400, -0.8), (40000, 96, 64, -2.0)])
def test_survivor_list_backward_edge_cases(P, W, H, scale_mu):
    """Survivor-driven backward on: partial panels and ragged images, huge splats (lists of one entry per quad for most
    tiles), and a small saturated image (long lists cut short by early termination: the lists end where the forward stopped)."""
    S, g = _case(P, W, H, seed=P + 1, scale_mu=scale_mu)
    dC, dI = _grads_in(H, W, 5)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)
    # a second backward through the predecessor kernel gives the same gradients up to the atomics' summation order
    old = _lib.set_option("composite_bwd", 3)
    try:
        grads3 = run_gpu(S, g, dC, dI)[4]
    finally:
        _lib.set_option("composite_bwd", old)
    for k in grads:
        sc = np.abs(grads3[k]).max() + 1e-20
        assert np.abs(grads[k] - grads3[k]).max() / sc < (5e-3 if k in ("scales", "rotations") else 2e-4), k


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("P,W,H", [(50000, 640, 480), (300, 48, 32), (5000, 1920, 1080)])
def test_sort_implementations_give_the_stock_order(impl, P, W, H):
    """Hand-written radix sort (1) and cub (0): identical, oracle-exact (tile, depth bits, index) order; sizes chosen to
    hit partial CTAs, > 1 scan chunk, and 13 tile bits (two passes) / 7 tile bits (one pass)."""
    S, g = _case(P, W, H, seed=P + impl, extent=1.1, scale_mu=-2.4)
    old = _lib.set_option("sort_impl", impl)
    try:
        color, radii, invd, state, _ = run_gpu(S, g)
    finally:
        _lib.set_option("sort_impl", old)
    st, _ = run_oracle(S, g)
    assert_forward_parity(st, color, radii, invd, state)


@pytest.mark.parametrize("bin_impl,sort_impl", [(1, 0), (1, 1), (0, 0)])
@pytest.mark.parametrize("P,W,H,scale_mu", [(50000, 640, 480, -2.4), (300, 48, 32, -2.4), (5000, 1920, 1080, -2.4), (400, 800, 608, -0.7)])
def test_binning_implementations_give_the_stock_order(bin_impl, sort_impl, P, W, H, scale_mu):
    """Cooperative counting binning (gms_binning.cuh, default) and the round-1 emit + radix-sort path: identical,
    oracle-exact (tile, depth bits, index) lists.  The last case has huge splats (rectangles of hundreds of tiles: the
    warp-cooperative branches) and long lists."""
    S, g = _case(P, W, H, seed=P + bin_impl, extent=1.1, scale_mu=scale_mu)
    old_b, old_s = _lib.set_option("bin_impl", bin_impl), _lib.set_option("sort_impl", sort_impl)
    try:
        color, radii, invd, state, _ = run_gpu(S, g)
    finally:
        _lib.set_option("bin_impl", old_b); _lib.set_option("sort_impl", old_s)
    st, _ = run_oracle(S, g)
    assert_forward_parity(st, color, radii, invd, state)


def _expected_flags(bin_impl, sort_impl, key16, T):
    """saved.flags bits 0 (counting binning ran) and 2 (16-bit tile keys).  The counting kernel needs two 32-bit rows of T
    counters plus 12 KB within the H100's 227 KB of opt-in shared memory per block; where they do not fit (T > 27518) the
    call falls back to emit + sort."""
    counting = bin_impl == 1 and 8 * T + 64 + 12288 <= 227 * 1024
    return int(counting) | (4 if not counting and sort_impl == 0 and key16 and T <= 65535 else 0)


def _nosync_call(S, g, cap):
    """gms_rasterize_forward_nosync through the raw C ABI with binning capacity `cap`; every scratch region carries a canary
    behind the bytes it asked for.  Returns (color, radii, invdepth, saved, n_host, debug state)."""
    import ctypes as C
    from types import SimpleNamespace
    from gms_b200 import rasterizer as R
    from gpu_helpers import gpu_settings
    dev = torch.device("cuda")
    W, H = S.image_width, S.image_height
    keep = []
    s = R._settings_struct(gpu_settings(S), dev, keep)
    t = {k: v.cuda().float().contiguous() for k, v in g.items()}
    P = t["means3D"].shape[0]
    i = R._inputs_struct(P, 16, t["means3D"], t["opacities"], t["shs"], None, t["scales"], t["rotations"], None)
    out_c = torch.full((3, H, W), -1.0, device=dev); out_r = torch.zeros(P, dtype=torch.int32, device=dev)
    out_d = torch.full((1, H, W), -1.0, device=dev)
    o = _lib.RasterOutputs(out_c.data_ptr(), out_r.data_ptr(), out_d.data_ptr())
    bufs, guard = {}, {}

    def _alloc(user, which, nbytes):
        b = torch.zeros(int(nbytes) + 4096, dtype=torch.uint8, device=dev)
        b[int(nbytes):] = 0xAB                              # canary behind the requested region
        bufs[int(which)] = b; guard[int(which)] = int(nbytes)
        return b.data_ptr()

    cb = _lib.ALLOC_FN(_alloc)
    saved = _lib.RasterSaved()
    n_host = torch.zeros(2, dtype=torch.int32).pin_memory()
    _lib.check(_lib.lib().gms_rasterize_forward_nosync(C.byref(s), C.byref(i), C.byref(o), cb, None, C.byref(saved), cap,
                                                       n_host.data_ptr(), torch.cuda.current_stream().cuda_stream), "nosync")
    torch.cuda.synchronize()
    for which, nb in guard.items():
        assert bool((bufs[which][nb:] == 0xAB).all()), f"scratch region {which} overrun"
    N = int(n_host[0])
    state = R.forward_debug_state(SimpleNamespace(bufs=bufs), min(N, cap), P, W, H, out_r,
                                  bin_state=(int(saved.binning_capacity), int(saved.flags)))
    return out_c.cpu().numpy(), out_r.cpu().numpy(), out_d.cpu().numpy(), saved, n_host, \
        {k: v.cpu().numpy() for k, v in state.items()}


@pytest.mark.parametrize("bin_impl", [0, 1])
def test_nosync_forward_matches_and_overflow_degrades_to_background(bin_impl):
    """gms_rasterize_forward_nosync at the capacity edges: N - 1 (overflow), N, N + 1 and N + 2*4096 + 1 (a sentinel tail
    longer than one CTA tile of the hand-written sort, and not a multiple of it).  With enough capacity the image and
    radii equal the synchronising call bit for bit, and the point list and tile ranges equal both the synchronising call and
    the oracle; N is reported through the mapped host word.  With too little, the overflow flag is raised and the frame
    renders the background.  No call writes past any scratch region.  Either binning, with the default sort (cub) and
    16-bit tile keys."""
    _nosync_with_options(bin_impl, 0, 1)


@pytest.mark.parametrize("bin_impl,sort_impl,key16", [(0, 0, 0), (0, 1, 1), (1, 1, 1)])
def test_nosync_capacity_edges_with_the_other_sorts_and_key_widths(bin_impl, sort_impl, key16):
    """The capacity edges of test_nosync_forward_matches_and_overflow_degrades_to_background for the remaining
    implementations: emit + cub sort on 32-bit keys, emit + hand-written sort (32-bit keys, device-side N), and the counting
    binning behind the hand-written depth sort."""
    _nosync_with_options(bin_impl, sort_impl, key16)


def _nosync_with_options(bin_impl, sort_impl, key16):
    S, g = _case(20000, 400, 300, seed=9)
    olds = {k: _lib.set_option(k, v) for k, v in (("bin_impl", bin_impl), ("sort_impl", sort_impl), ("key16", key16))}
    try:
        _nosync_body(S, g, _expected_flags(bin_impl, sort_impl, key16, 25 * 19))
    finally:
        for k, v in olds.items():
            _lib.set_option(k, v)


def _nosync_body(S, g, flags):
    color, radii, invd, state, _ = run_gpu(S, g)
    N = state["num_rendered"]
    st, _ = run_oracle(S, g)
    np.testing.assert_array_equal(state["point_list"].astype(np.uint32), st.point_list)
    np.testing.assert_array_equal(state["ranges"], st.ranges)
    for cap, expect_overflow in ((N - 1, True), (N, False), (N + 1, False), (N + 2 * 4096 + 1, False)):
        out_c, out_r, out_d, saved, n_host, ns = _nosync_call(S, g, cap)
        assert int(saved.num_rendered) == -1 and (int(saved.flags) & 5) == flags and int(saved.binning_capacity) == cap
        assert int(n_host[0]) == N and int(n_host[1]) == int(expect_overflow), (cap, N, int(n_host[0]), int(n_host[1]))
        np.testing.assert_array_equal(out_r, radii)
        if expect_overflow:
            bg = np.asarray(S.bg, np.float32)
            assert np.array_equal(out_c, np.broadcast_to(bg[:, None, None], out_c.shape)) and float(np.abs(out_d).max()) == 0.0
        else:
            np.testing.assert_array_equal(ns["point_list"], state["point_list"], err_msg=f"capacity {cap}")
            np.testing.assert_array_equal(ns["ranges"], state["ranges"], err_msg=f"capacity {cap}")
            np.testing.assert_array_equal(out_c, color); np.testing.assert_array_equal(out_d, invd)


@pytest.mark.parametrize("bin_impl,sort_impl", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("W,H", [(4080, 4112), (4096, 4096)])
def test_nosync_binning_at_the_16_32_bit_key_boundary(W, H, bin_impl, sort_impl):
    """T = 255 x 257 = 65535 tiles, the largest grid on 16-bit tile keys (ids up to 65534, sentinel 0xFFFF; the hand-written
    sort takes two 8-bit passes), and T = 256 x 256 = 65536 on 32-bit keys (three hand-written passes).  Forward only:
    the sync-free call gives the synchronising call's image bit for bit and the oracle's point list and tile ranges; the
    image matches the oracle's composite on every 97th tile."""
    from oracle import raster
    S, g = _case(3000, W, H, seed=W, extent=1.1, scale_mu=-3.2)
    T = (W // 16) * (H // 16)
    olds = {k: _lib.set_option(k, v) for k, v in (("bin_impl", bin_impl), ("sort_impl", sort_impl))}
    try:
        color, radii, invd, state, _ = run_gpu(S, g)
        N = state["num_rendered"]
        out_c, out_r, out_d, saved, n_host, ns = _nosync_call(S, g, N + 2 * 4096 + 1)
    finally:
        for k, v in olds.items():
            _lib.set_option(k, v)
    assert (int(saved.flags) & 5) == _expected_flags(bin_impl, sort_impl, 1, T)
    assert int(n_host[0]) == N and int(n_host[1]) == 0
    np.testing.assert_array_equal(out_r, radii)
    np.testing.assert_array_equal(out_c, color); np.testing.assert_array_equal(out_d, invd)
    st = raster.preprocess(S, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    np.testing.assert_array_equal(radii, st.radii)
    raster.bin_tiles(st)
    assert st.N == N and st.ranges.shape[0] == T
    for what in (state, ns):
        np.testing.assert_array_equal(what["point_list"].astype(np.uint32), st.point_list)
        np.testing.assert_array_equal(what["ranges"], st.ranges)
    raster.set_tile_stride(97)
    try:
        raster.composite(st)
    finally:
        raster.set_tile_stride(1)
    gx, worst, amb = W // 16, 0.0, 0
    for tile in range(0, T, 97):
        x0, y0 = (tile % gx) * 16, (tile // gx) * 16
        sl = (slice(None), slice(y0, y0 + 16), slice(x0, x0 + 16))
        ok = st.ambiguous[sl[1:]] == 0
        amb += int((~ok).sum())
        worst = max(worst, float(np.abs(out_c[sl] - st.color[sl])[:, ok].max()) if ok.any() else 0.0)
    print(f"[key boundary] {W}x{H} T={T} N={N} flags={int(saved.flags)} sampled tiles={len(range(0, T, 97))} "
          f"ambiguous px={amb} max|image-oracle|={worst:.2e}")
    assert worst <= 1e-5


@pytest.mark.parametrize("P,deg", [(4001, 3), (77, 1), (12345, 0)])
def test_sh_tile_staging_equals_direct_access(P, deg):
    """Option "sh_staged": SH rows (and their gradient rows) through the per-warp shared-memory tile vs per-lane global
    accesses.  Same arithmetic: colours and radii are bit-identical, dL/dshs agrees to the run-to-run noise of the upstream
    atomics, with exactly zero rows for culled Gaussians and a last warp that is only partly inside P."""
    S, g = _case(P, 200, 152, seed=P, sh_degree=deg, extent=2.5)      # extent 2.5: a good share of the splats is culled
    dC, dI = _grads_in(152, 200, 9)
    res = []
    default = _lib.set_option("sh_staged", 2)
    try:
        for staged in (2, 1, 0):      # 2: gradient rows computed in place in the tile; 1: register copies; 0: direct
            _lib.set_option("sh_staged", staged)
            res.append(run_gpu(S, g, dC, dI))
    finally:
        _lib.set_option("sh_staged", default)
    a = res[0]
    for b in res[1:]:
        np.testing.assert_array_equal(a[0], b[0]); np.testing.assert_array_equal(a[1], b[1])
        # dL/dshs = basis * dL/dcolour: the colour gradient comes out of composite_bwd's float atomics, so runs differ in
        # the last bits; the staging itself adds no arithmetic
        scale = np.abs(a[4]["shs"]).max()
        np.testing.assert_allclose(a[4]["shs"], b[4]["shs"], rtol=0, atol=2e-5 * scale)
        np.testing.assert_array_equal(a[4]["shs"] == 0, b[4]["shs"] == 0)
    assert (a[1] == 0).any() and (a[1] > 0).any()
    assert np.abs(a[4]["shs"][a[1] == 0]).max() == 0.0
    st, gref = run_oracle(S, g, dC, dI)
    assert_forward_parity(st, a[0], a[1], a[2], a[3])
    # extent 2.5 puts splats next to the camera: screen-filling footprints whose gradients are fp32 atomic sums over
    # ~1e4 pixels with cancellation (the oracle sums in double) -- 5x the usual tolerance for this scene
    assert_grad_parity(a[4], gref, tol=1e-3)


def test_empty_and_invisible_inputs():
    S, g = _case(10, 64, 64, seed=1)
    e = {k: v[:0] for k, v in g.items()}
    color, radii, invd, state, _ = run_gpu(S, e)
    assert radii.shape == (0,) and np.allclose(color, np.float32([0.1, 0.4, 0.8])[:, None, None]) and (invd == 0).all()
    far = dict(g); far["means3D"] = g["means3D"] + torch.tensor([100.0, 0, 0])
    dC, dI = _grads_in(64, 64, 1)
    color, radii, invd, state, grads = run_gpu(S, far, dC, dI)
    assert (radii == 0).all() and state["num_rendered"] == 0
    assert all(np.abs(v).max() == 0 for v in grads.values())


def test_forward_is_deterministic():
    S, g = _case(20000, 320, 240, seed=10)
    a = run_gpu(S, g); b = run_gpu(S, g)
    np.testing.assert_array_equal(a[0], b[0]); np.testing.assert_array_equal(a[3]["point_list"], b[3]["point_list"])


def test_mark_visible():
    import diff_gaussian_rasterization as dgr
    from gpu_helpers import gpu_settings
    from oracle import raster
    S, g = _case(5000, 64, 64, seed=12, extent=6.0)
    r = dgr.GaussianRasterizer(raster_settings=gpu_settings(S))
    vis = r.markVisible(g["means3D"].cuda())
    np.testing.assert_array_equal(vis.cpu().numpy(), raster.mark_visible(S, g["means3D"]))
