"""GPU: the per-match evaluation statistics (csrc/match_stats.cu via pdc_b200.evaluation) against the executed reference's
fixture (tests/golden/match_statistics.npz) and the float64 oracle (oracle/match_stats_oracle.py).

Gates: counts and pixel indices exact; float32 columns bit-equal (norm_diff_descriptor_ground_truth within 2 ulp of the
reference's np.linalg.norm); float64 columns within 1e-12 relative; NaN in the same places."""
import os

import numpy as np
import pytest
import torch

import pdc_b200
from pdc_b200 import evaluation as E
from oracle import match_stats_oracle as MO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "match_statistics.npz")
INTS = ["u_pred", "v_pred", "u_pred_masked", "v_pred_masked", "num_pixels_closer_than_ground_truth",
        "num_pixels_closer_than_ground_truth_masked", "num_pixels_in_masked_image"]


def _f64_close(got, ref, rel=1e-12):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    err = np.abs(got[ok] - ref[ok]) / np.maximum(np.abs(ref[ok]), 1e-300)
    err[np.abs(got[ok] - ref[ok]) <= 1e-15] = 0.0
    return float(err.max()) if err.size else 0.0


def _run(res_a, res_b, uv_a, uv_b, pair, mask, da, db, pa, pb, K):
    t = lambda x, dt=torch.float32: torch.as_tensor(np.asarray(x)).to(DEV, dt)
    out = E.match_statistics(t(res_a), t(res_b), t(uv_a, torch.int64), t(uv_b, torch.int64), t(pair, torch.int64), t(mask), t(da), t(db),
                             pa, pb, K)
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("D", [3, 9])
def test_golden_cases_equal_the_executed_reference(D):
    g = np.load(GOLDEN)
    ra = g["res_a_d%d" % D].astype(np.float32); rb = g["res_b_d%d" % D].astype(np.float32)
    uv_a = g["uv_a_d%d" % D]; uv_b = g["uv_b_d%d" % D]
    Q = len(uv_a)
    N = 3                                              # object mask, full mask, empty mask: one launch
    pair = np.repeat(np.arange(N), Q)
    rep = lambda x: np.repeat(x[None], N, 0)
    got = _run(rep(ra), rep(rb), np.tile(uv_a, (N, 1)), np.tile(uv_b, (N, 1)), pair, g["mask_b"], rep(g["depth_a"]),
               rep(g["depth_b"]), rep(g["pose_a"]), rep(g["pose_b"]), g["K"])
    assert int(got["bad_queries"][0]) == 0
    worst = 0.0
    for n in range(N):
        sl = slice(n * Q, (n + 1) * Q)
        raised = g["out_d%d_p%d/raised" % (D, n)]
        ref = lambda c: g["out_d%d_p%d/%s" % (D, n, c)]
        if n == 2:
            assert (raised == "ZeroDivisionError").all() and np.isnan(got["fraction_pixels_closer_than_ground_truth_masked"][sl]).all()
            assert (got["num_pixels_in_masked_image"][sl] == 0).all()
            # the reference raises before its row is complete; every other column follows its float64 statements, so the
            # masked minimum nd + 1e6 is float64 (in float32 its ulp would be 0.0625)
            for i in range(Q):
                o = MO.one_match(g["depth_a"], g["depth_b"], g["mask_b"][n], tuple(uv_a[i]), tuple(uv_b[i]), g["pose_a"],
                                 g["pose_b"], ra, rb, g["K"], empty_mask_nan=True)
                for c in E.F64_COLUMNS:
                    assert _f64_close(got[c][n * Q + i:n * Q + i + 1], [o[c]]) <= 1e-12, (i, c)
                assert got["norm_diff_descriptor_masked"][n * Q + i] == o["norm_diff_descriptor_masked"]
            continue
        assert np.array_equal(got["norm_diff_descriptor"][sl], ref("norm_diff_descriptor"))
        gt, rt = got["norm_diff_descriptor_ground_truth"][sl], ref("norm_diff_descriptor_ground_truth")
        assert (np.abs(gt.view(np.int32) - rt.view(np.int32)) <= 2).all()
        assert np.array_equal(got["is_valid"][sl], ref("is_valid") == 1)
        assert np.array_equal(got["is_valid_masked"][sl], ref("is_valid_masked") == 1)
        for c in E.F64_COLUMNS:
            e = _f64_close(got[c][sl], ref(c))
            assert e <= 1e-12, (c, e)
            worst = max(worst, e)
    print("golden D=%d: worst float64 relative error %.3g" % (D, worst))
    # the reference-signature wrapper: one row, and ZeroDivisionError on the empty mask
    DCE = E.DenseCorrespondenceEvaluation
    args = lambda n, i: (g["depth_a"], g["depth_b"], None, g["mask_b"][n], tuple(uv_a[i]), tuple(uv_b[i]), g["pose_a"], g["pose_b"],
                         ra, rb, g["K"])
    row = DCE.compute_descriptor_match_statistics(*args(0, 4)).dataframe
    for c in E.F32_COLUMNS + E.F64_COLUMNS:
        assert _f64_close(row[c].values, g["out_d%d_p0/%s" % (D, c)][4:5]) <= 1e-12, c
    with pytest.raises(ZeroDivisionError):
        DCE.compute_descriptor_match_statistics(*args(2, 0))


def _scene(rng, N, H, W, D, Q):
    """N random pairs; descriptors as the permuted [H,W,D] views forward_single_image_tensor returns."""
    a = torch.from_numpy(rng.standard_normal((N, D, H, W)).astype(np.float32)).to(DEV)
    b = torch.from_numpy(rng.standard_normal((N, D, H, W)).astype(np.float32)).to(DEV)
    res_a, res_b = a.permute(0, 2, 3, 1), b.permute(0, 2, 3, 1)
    mask = (rng.random((N, H, W)) < 0.6).astype(np.float32)
    if N > 1:
        mask[0] = 0          # an empty mask: every masked distance is nd + 1e6, whose float64 rounding the columns show
    da = rng.integers(0, 3000, (N, H, W)).astype(np.float32); db = rng.integers(0, 12000, (N, H, W)).astype(np.float32)
    da[rng.random((N, H, W)) < 0.1] = 0; db[rng.random((N, H, W)) < 0.1] = 0
    pair = np.sort(rng.integers(0, N, Q))
    uv_a = np.stack([rng.integers(0, W, Q), rng.integers(0, H, Q)], 1)
    uv_b = np.stack([rng.integers(0, W, Q), rng.integers(0, H, Q)], 1)
    K = np.array([[533.6, 0, W / 2.0 - 0.4], [0, 534.7, H / 2.0 + 0.3], [0, 0, 1.0]])
    poses = lambda: np.stack([np.vstack([np.hstack([np.linalg.qr(rng.standard_normal((3, 3)))[0], rng.standard_normal((3, 1))]),
                                         [0, 0, 0, 1]]) for _ in range(N)])
    return res_a, res_b, uv_a, uv_b, pair, mask, da, db, poses(), poses(), K


def _device(s):
    res_a, res_b, uv_a, uv_b, pair, mask, da, db, pa, pb, K = s
    t = lambda x, dt=torch.float32: torch.as_tensor(np.asarray(x)).to(DEV, dt)
    out = E.match_statistics(res_a, res_b, t(uv_a, torch.int64), t(uv_b, torch.int64), t(pair, torch.int64), t(mask), t(da), t(db),
                             pa, pb, K)
    return {k: v.cpu().numpy() for k, v in out.items()}


RANDOM = [(1, 480, 640, 3, 100), (1, 480, 640, 16, 40), (2, 37, 53, 1, 50), (3, 7, 13, 7, 30), (2, 61, 45, 8, 64),
          (4, 33, 29, 9, 70), (2, 40, 56, 17, 40), (2, 24, 20, 32, 33), (100, 24, 32, 3, 1000)]


@pytest.mark.parametrize("N,H,W,D,Q", RANDOM)
def test_random_cases_against_the_oracle(N, H, W, D, Q):
    rng = np.random.default_rng(1000 * D + Q)
    s = _scene(rng, N, H, W, D, Q)
    got = _device(s)
    res_a, res_b = s[0].cpu().numpy(), s[1].cpu().numpy()
    ref = MO.match_statistics(res_a, res_b, *s[2:], threshold="device")
    assert np.array_equal(got["norm_diff_descriptor"], ref["norm_diff_descriptor"])              # numpy's find_best_match
    assert np.array_equal(got["norm_diff_descriptor_ground_truth"], ref["norm_diff_descriptor_ground_truth"])
    for c in INTS:
        assert np.array_equal(got[c], ref[c]), c
    assert np.array_equal(got["is_valid"], ref["is_valid"]) and np.array_equal(got["is_valid_masked"], ref["is_valid_masked"])
    worst = max(_f64_close(got[c], ref[c]) for c in E.F64_COLUMNS)
    assert worst <= 1e-12, worst
    # each count lies between the counts at nd(uv_b) and at the reference's np.linalg.norm threshold
    refl = MO.match_statistics(res_a, res_b, *s[2:], threshold="reference")
    for c in ("num_pixels_closer_than_ground_truth", "num_pixels_closer_than_ground_truth_masked"):
        lo, hi = np.minimum(ref[c], refl[c]), np.maximum(ref[c], refl[c])
        assert ((lo <= got[c]) & (got[c] <= hi)).all()
    gt, rt = got["norm_diff_descriptor_ground_truth"], refl["norm_diff_descriptor_ground_truth"]
    print("N %d %dx%d D %d Q %d: worst float64 rel %.3g, threshold vs np.linalg.norm max %d ulp" % (
        N, H, W, D, Q, worst, int(np.abs(gt.view(np.int32) - rt.view(np.int32)).max())))


def test_batched_equals_per_pair_and_repeats_bit_identically():
    rng = np.random.default_rng(7)
    N, H, W, D, Q = 3, 48, 64, 16, 45
    s = _scene(rng, N, H, W, D, Q)
    s = s[:4] + (rng.permutation(s[4]),) + s[5:]          # pairs interleaved: no block sees a single pair
    full = _device(s)
    again = _device(s)
    for k in full:
        assert np.array_equal(full[k].view(np.uint8), again[k].view(np.uint8)), k
    res_a, res_b, uv_a, uv_b, pair, mask, da, db, pa, pb, K = s
    for n in range(N):
        sel = np.nonzero(pair == n)[0]
        one = _device((res_a[n], res_b[n], uv_a[sel], uv_b[sel], np.zeros(len(sel), np.int64), mask[n], da[n], db[n], pa[n:n + 1],
                       pb[n:n + 1], K))
        for k in one:
            if k != "bad_queries":
                assert np.array_equal(one[k], full[k][sel], equal_nan=True), (n, k)


def test_out_of_range_queries_get_nan_rows():
    rng = np.random.default_rng(3)
    s = list(_scene(rng, 2, 20, 30, 3, 6))
    s[4] = np.array([0, 0, 1, 2, -1, 1]); s[2] = s[2].copy(); s[2][1] = (30, 0); s[3] = s[3].copy(); s[3][5] = (0, 20)
    got = _device(tuple(s))
    bad = np.array([False, True, False, True, True, True])
    assert int(got["bad_queries"][0]) == 4
    assert np.isnan(got["norm_diff_descriptor"][bad]).all() and np.isnan(got["pixel_match_error_l2"][bad]).all()
    assert (got["u_pred"][bad] == -1).all() and not np.isnan(got["norm_diff_descriptor"][~bad]).any()
    # a pair whose descriptor image B is all NaN has no masked minimum: its queries get the same rows, nothing is read
    s = list(_scene(rng, 2, 20, 30, 3, 6))
    s[4] = np.array([0, 0, 0, 1, 1, 1]); s[1] = s[1].clone(); s[1][1] = float("nan")
    got = _device(tuple(s))
    assert int(got["bad_queries"][0]) == 3 and (got["u_pred_masked"][3:] == -1).all() and (got["u_pred_masked"][:3] >= 0).all()


def test_wrapper_refuses_wrong_dtypes_and_shapes():
    H, W, D = 8, 12, 3
    r = torch.zeros(1, H, W, D, device=DEV)
    i2 = torch.zeros(1, 2, dtype=torch.int64, device=DEV); p = torch.zeros(1, dtype=torch.int64, device=DEV)
    m = torch.ones(1, H, W, device=DEV)
    pose = np.eye(4)[None]
    call = lambda **kw: E.match_statistics(*[kw.get(k, v) for k, v in (("ra", r), ("rb", r), ("ua", i2), ("ub", i2), ("p", p),
                                                                        ("m", m), ("da", m), ("db", m))], pose, pose, np.eye(3))
    with pytest.raises(RuntimeError, match="float32"):
        call(ra=r.double())
    with pytest.raises(RuntimeError, match="int64"):
        call(ua=i2.int())
    with pytest.raises(RuntimeError, match="shape"):
        call(ub=torch.zeros(1, 3, dtype=torch.int64, device=DEV))
    with pytest.raises(RuntimeError, match="shape"):
        call(m=torch.ones(1, H + 1, W, device=DEV))
    with pytest.raises(RuntimeError, match="same shape"):
        call(rb=torch.zeros(1, H, W, D + 1, device=DEV))
    with pytest.raises(RuntimeError, match="descriptor dimension"):
        z = torch.zeros(1, H, W, 33, device=DEV); call(ra=z, rb=z)


def test_quantitative_analysis_on_pair_end_to_end():
    """Resnet34_8s in eval mode on the synthetic plane scene of tests/test_gpu_ops.py; the rows equal the oracle's on the
    same descriptor images (copied to the host) and the same chosen matches."""
    H, W, D = 480, 640, 3
    K = np.array([[533.6422696034836, 0, 319.4091030774892], [0, 534.7824445233571, 236.4374299691866], [0, 0, 1.0]])

    def pose(rx, ry, t):
        cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
        Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        T = np.eye(4); T[:3, :3] = Ry.dot(Rx); T[:3, 3] = t
        return T
    pose_a = pose(0.02, -0.03, [0.0, 0.0, 0.0]); pose_b = pose(-0.05, 0.12, [0.18, -0.04, 0.05])

    def render(T):
        us, vs = np.meshgrid(np.arange(W), np.arange(H))
        rays = np.linalg.inv(K).dot(np.stack([us.ravel(), vs.ravel(), np.ones(H * W)]))
        rw = T[:3, :3].dot(rays); o = T[:3, 3]
        nrm = np.array([-0.1, 0.05, 1.0]); d0 = 1.2
        return ((d0 - nrm.dot(o)) / nrm.dot(rw) * 1000.0).reshape(H, W)
    depth_a = np.round(render(pose_a)).astype(np.uint16); depth_b = np.round(render(pose_b)).astype(np.uint16)
    depth_a[200:230, 300:340] = 0; depth_b[100:260, 380:470] = 600
    mask_a = np.zeros((H, W), np.uint8); mask_a[100:400, 150:500] = 1
    mask_b = np.zeros((H, W), np.uint8); mask_b[80:420, 120:540] = 1
    dcn = pdc_b200.DenseCorrespondenceNetwork.from_config({"descriptor_dimension": D, "image_width": W, "image_height": H},
                                                           load_stored_params=False)
    dcn.eval()
    gen = torch.Generator().manual_seed(5)
    rgb_a = torch.randn(3, H, W, generator=gen); rgb_b = torch.randn(3, H, W, generator=gen)
    g = torch.Generator(device=DEV).manual_seed(11)
    rows = E.quantitative_analysis_on_pair(dcn, rgb_a, rgb_b, depth_a, depth_b, mask_a, mask_b, pose_a, pose_b, K, num_matches=100,
                                           generator=g, num_attempts=400)
    assert rows is not None and 50 <= len(rows["uv_a"]) <= 100
    with torch.no_grad():
        res_a = dcn.forward_single_image_tensor(rgb_a).cpu().numpy()[None]
        res_b = dcn.forward_single_image_tensor(rgb_b).cpu().numpy()[None]
    M = len(rows["uv_a"])
    ref = MO.match_statistics(res_a, res_b, rows["uv_a"], rows["uv_b"], np.zeros(M, np.int64), mask_b[None], depth_a[None],
                              depth_b[None], pose_a[None], pose_b[None], K, threshold="device")
    for c in E.F32_COLUMNS + INTS + ["is_valid", "is_valid_masked"]:
        assert np.array_equal(rows[c], ref[c]), c
    assert max(_f64_close(rows[c], ref[c]) for c in E.F64_COLUMNS) <= 1e-12
