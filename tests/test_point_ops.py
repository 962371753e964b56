"""Farthest point sampling and ball query (pytorch3d_b200.point_ops, DESIGN.md section 22).

CPU: a numpy restatement of the two kernels' contracts (`fps_restated`, `ball_restated`, the float64 `ball_grad_restated`)
matches the records of the reference's CPU ops (tests/golden/make_point_ops_golden.py); host-side errors; D != 3;
`install_point_ops()` routing with stand-in pytorch3d modules.
GPU: sampled indices, idx and dists bit for bit the reference's CUDA kernels recompiled for sm_90a
(oracle/_ref/ref_point_ops_cuda.so), nn bitwise masked_gather(p2, idx), gradients per element against the float64
restatement and within tolerance of the reference's chain, determinism, host synchronisations, peak memory, argument
checks and one PointNet++ set-abstraction step.

The restatements are written from the contract: pair distances are the FFMA chain fma(dz, dz, fma(dy, dy, fma(dx, dx,
0))) in float32 (formed here in float64, exact for the small-integer scenes the records use), FPS's running distance
starts at 1e10 and is lowered by fmin, its selection is the first maximum, and ball query keeps the first K targets
with dist2 < float32(r) * float32(r).
"""
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

from helpers import GOLDEN_DIR

DEV = "cuda"
GOLDEN = os.path.join(GOLDEN_DIR, "reference_golden_point_ops.npz")


# ---- restatements -------------------------------------------------------------------------------------------------

def sqdist(a, b):
    """fma(dz, dz, fma(dy, dy, fma(dx, dx, 0))) with d = a - b in float32, broadcast over leading dimensions."""
    with np.errstate(invalid="ignore", over="ignore"):
        d = (np.asarray(a, np.float32) - np.asarray(b, np.float32)).astype(np.float64)
        acc = (d[..., 0] * d[..., 0]).astype(np.float32)
        acc = (d[..., 1] * d[..., 1] + acc).astype(np.float32)
        return (d[..., 2] * d[..., 2] + acc).astype(np.float32)


def _clamp_len(lengths, n, P):
    return P if lengths is None else int(min(max(int(lengths[n]), 0), P))


def fps_restated(points, lengths, K, start, max_K):
    points = np.asarray(points, np.float32)
    N, P, _ = points.shape
    idx = np.full((N, max_K), -1, np.int64)
    if max_K == 0 or P == 0:
        return idx
    for n in range(N):
        L, s = _clamp_len(lengths, n, P), int(start[n])
        if L > 0 and not 0 <= s < L:
            continue  # a start outside the cloud selects nothing
        idx[n, 0] = s
        kn = min(int(K[n]), L, max_K)
        d = np.full(L, 1e10, np.float32)
        for k in range(1, kn):
            d = np.fmin(sqdist(points[n, s], points[n, :L]), d)
            s = int(np.argmax(d))
            idx[n, k] = s
    return idx


def ball_restated(p1, p2, lengths1, lengths2, K, radius, skip):
    p1, p2 = np.asarray(p1, np.float32), np.asarray(p2, np.float32)
    N, P1, _ = p1.shape
    P2 = p2.shape[1]
    r = np.float32(radius)
    r2 = np.float32(r * r)
    idx = np.full((N, P1, K), -1, np.int64)
    dists = np.zeros((N, P1, K), np.float32)
    if skip and r < 0:
        return idx, dists
    for n in range(N):
        L1, L2 = _clamp_len(lengths1, n, P1), _clamp_len(lengths2, n, P2)
        for i in range(L1):
            d = sqdist(p1[n, i], p2[n, :L2])
            hits = np.nonzero(d < r2)[0][:K]
            idx[n, i, :len(hits)] = hits
            dists[n, i, :len(hits)] = d[hits]
    return idx, dists


def ball_grad_restated(p1, p2, idx, g_dists, g_nn):
    """float64 knn_points_backward(norm=2) plus masked_gather's backward."""
    p1, p2 = np.asarray(p1, np.float64), np.asarray(p2, np.float64)
    gp1, gp2 = np.zeros_like(p1), np.zeros_like(p2)
    n, i, k = np.nonzero(idx >= 0)
    j = idx[n, i, k]
    with np.errstate(invalid="ignore"):
        if g_dists is not None:
            diff = 2.0 * np.asarray(g_dists, np.float64)[n, i, k][:, None] * (p1[n, i] - p2[n, j])
            np.add.at(gp1, (n, i), diff)
            np.add.at(gp2, (n, j), -diff)
        if g_nn is not None:
            np.add.at(gp2, (n, j), np.asarray(g_nn, np.float64)[n, i, k])
    return gp1, gp2


# ---- scenes (shared with tests/golden/make_point_ops_golden.py) ---------------------------------------------------

def fps_scenes():
    """name -> dict(points, lengths, K (list), start, max_K); small-integer coordinates, so ties are common and the
    reference's CPU and CUDA arithmetic agree."""
    g = torch.Generator().manual_seed(22)
    s = {}
    s["uniform"] = dict(points=torch.randint(-4, 5, (3, 40, 3), generator=g).float(), lengths=None, K=[10, 10, 10])
    s["ragged"] = dict(points=torch.randint(-3, 4, (4, 40, 3), generator=g).float(), lengths=[40, 17, 5, 1],
                       K=[0, 1, 30, 12])
    dup = torch.randint(-2, 3, (2, 6, 3), generator=g).float().repeat(1, 4, 1)
    s["duplicates"] = dict(points=dup, lengths=[24, 13], K=[20, 20])
    s["k1"] = dict(points=torch.randint(-4, 5, (2, 9, 3), generator=g).float(), lengths=None, K=[1, 1])
    s["grid"] = dict(points=torch.stack(torch.meshgrid(*[torch.arange(4.0)] * 3, indexing="ij"), -1).reshape(1, 64, 3),
                     lengths=None, K=[64])
    for v in s.values():
        v["start"] = [0] * v["points"].shape[0]
    # random starts: the reference's expressions, recorded
    gr = torch.Generator().manual_seed(5)
    s["random_ragged"] = dict(points=torch.randint(-4, 5, (3, 30, 3), generator=g).float(), lengths=[30, 21, 7],
                              K=[8, 8, 8])
    s["random_ragged"]["start"] = (torch.tensor([30, 21, 7]) * torch.rand(3, generator=gr)).to(torch.int64).tolist()
    s["random_full"] = dict(points=torch.randint(-4, 5, (3, 30, 3), generator=g).float(), lengths=None, K=[8, 8, 8])
    s["random_full"]["start"] = torch.randint(high=30, size=(3,), generator=gr).tolist()
    for v in s.values():
        v["max_K"] = max(v["K"])
    return s


BALL_CASES = {  # name -> (scene, K, radius, skip)
    "k1": ("uniform", 1, 1.5, False), "k32": ("uniform", 32, 1.5, False), "k500": ("uniform", 500, 5.0, False),
    "k_above_p2": ("uniform", 60, 100.0, False), "on_radius": ("uniform", 32, 2.0, False),
    "all_hit": ("uniform", 50, 100.0, True), "none_hit": ("uniform", 8, 0.0, False),
    "skip": ("uniform", 32, 1.5, True), "ragged": ("ragged", 16, 1.5, False),
    "negative_radius": ("uniform", 16, -1.5, False), "negative_radius_skip": ("uniform", 16, -1.5, True),
    "nonfinite": ("nonfinite", 16, 2.5, False), "nonfinite_skip": ("nonfinite", 16, 2.5, True),
}


def ball_scenes():
    """name -> dict(p1, p2, lengths1, lengths2); small-integer coordinates (squared distances are integers, so radius
    2 puts points exactly on the sphere)."""
    g = torch.Generator().manual_seed(23)
    s = {}
    s["uniform"] = dict(p1=torch.randint(-3, 4, (2, 30, 3), generator=g).float(),
                        p2=torch.randint(-3, 4, (2, 50, 3), generator=g).float(), lengths1=None, lengths2=None)
    s["ragged"] = dict(p1=torch.randint(-3, 4, (3, 20, 3), generator=g).float(),
                       p2=torch.randint(-3, 4, (3, 25, 3), generator=g).float(), lengths1=[20, 7, 0],
                       lengths2=[25, 0, 9])
    p1 = torch.randint(-2, 3, (1, 12, 3), generator=g).float()
    p2 = torch.randint(-2, 3, (1, 20, 3), generator=g).float()
    p1[0, 2, 1] = float("nan")
    p1[0, 5, 0] = float("inf")
    p2[0, 3, 2] = float("nan")
    p2[0, 7, 1] = float("-inf")
    s["nonfinite"] = dict(p1=p1, p2=p2, lengths1=None, lengths2=None)
    return s


def ball_upstream(name, idx_shape):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    return (torch.randint(-3, 4, idx_shape, generator=g).float() / 4,
            torch.randint(-3, 4, idx_shape + (3,), generator=g).float() / 4)


def _np(x):
    return None if x is None else np.asarray(x)


@pytest.fixture(scope="module")
def golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/reference_golden_point_ops.npz missing")
    return np.load(GOLDEN)


# ---- CPU: the restatements against the records --------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(fps_scenes()))
def test_fps_restated_matches_record(golden, name):
    sc = fps_scenes()[name]
    got = fps_restated(sc["points"].numpy(), _np(sc["lengths"]), sc["K"], sc["start"], sc["max_K"])
    assert np.array_equal(golden["fps/%s/0/start" % name], np.asarray(sc["start"]))
    np.testing.assert_array_equal(got, golden["fps/%s/0/idx" % name])


def test_fps_records_cover_the_contract(golden):
    ragged = golden["fps/ragged/0/idx"]
    assert list(ragged[0]) == [0] + [-1] * 29          # K = 0 still writes the start
    assert list(ragged[1]) == [0] + [-1] * 29          # K = 1
    assert (ragged[2, :5] >= 0).all() and (ragged[2, 5:] == -1).all()  # K above the length
    dup = golden["fps/duplicates/0/idx"][0]
    assert len(set(dup.tolist())) < len(dup)           # fewer distinct points than K repeats indices


def test_fps_restated_empty_and_nonfinite():
    # empty clouds and out-of-range starts: the documented rows
    pts = np.zeros((3, 5, 3), np.float32)
    got = fps_restated(pts, [0, 5, 3], [3, 3, 3], [0, 7, -1], 3)
    assert got.tolist() == [[0, -1, -1], [-1, -1, -1], [-1, -1, -1]]
    # a NaN point keeps the initial 1e10 (fmin ignores NaN) and is selected again; inf likewise through inf - inf
    pts = np.array([[[0, 0, 0], [1, 0, 0], [np.nan, 0, 0], [3, 0, 0]]], np.float32)
    assert fps_restated(pts, None, [4], [0], 4).tolist() == [[0, 2, 2, 2]]
    pts = np.array([[[0, 0, 0], [2, 0, 0], [np.inf, 0, 0]]], np.float32)
    assert fps_restated(pts, None, [3], [0], 3).tolist() == [[0, 2, 2]]
    pts = np.array([[[0, 0, 0], [1e6, 0, 0], [-1e6, 0, 0], [1, 0, 0]]], np.float32)  # distances above the 1e10 cap tie
    assert fps_restated(pts, None, [3], [0], 3).tolist() == [[0, 1, 2]]


@pytest.mark.parametrize("case", sorted(BALL_CASES))
def test_ball_restated_matches_record(golden, case):
    scene, K, radius, skip = BALL_CASES[case]
    sc = ball_scenes()[scene]
    idx, dists = ball_restated(sc["p1"].numpy(), sc["p2"].numpy(), _np(sc["lengths1"]), _np(sc["lengths2"]), K,
                               radius, skip)
    np.testing.assert_array_equal(idx, golden["ball/%s/0/idx" % case])
    assert np.array_equal(dists.view(np.int32), golden["ball/%s/0/dists" % case].view(np.int32))


def test_ball_records_cover_the_contract(golden):
    assert (golden["ball/none_hit/0/idx"] == -1).all()
    assert (golden["ball/negative_radius_skip/0/idx"] == -1).all()
    assert (golden["ball/negative_radius/0/idx"] >= 0).any()        # dist2 < r^2 without the cube test
    assert (golden["ball/all_hit/0/idx"][:, :, :50] >= 0).all()
    assert (golden["ball/k_above_p2/0/idx"][:, :, 50:] == -1).all()
    assert (golden["ball/k500/0/idx"] >= 0).sum(-1).max() > 32
    assert (golden["ball/on_radius/0/dists"] < 4).all()            # dist2 = 4 = r^2 is outside
    sc = ball_scenes()["uniform"]
    d = sqdist(sc["p1"].numpy()[:, :, None], sc["p2"].numpy()[:, None])
    assert (d == 4).any()


@pytest.mark.parametrize("case", ["k32", "k500", "ragged", "nonfinite"])
def test_ball_grad_restated_matches_record(golden, case):
    scene, K, radius, skip = BALL_CASES[case]
    sc = ball_scenes()[scene]
    idx = golden["ball/%s/0/idx" % case]
    gd, gnn = ball_upstream(case, idx.shape)
    gp1, gp2 = ball_grad_restated(sc["p1"].numpy(), sc["p2"].numpy(), idx, gd.numpy(), gnn.numpy())
    with np.errstate(invalid="ignore"):
        np.testing.assert_allclose(gp1, golden["ball/%s/0/grad_p1" % case], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(gp2, golden["ball/%s/0/grad_p2" % case], rtol=1e-6, atol=1e-6)


# ---- CPU: host-side errors and routing -----------------------------------------------------------------------------

def test_host_errors_cpu():
    from pytorch3d_b200 import point_ops as po
    x = torch.zeros(2, 5, 3)
    with pytest.raises(ValueError, match="points and lengths must have same batch dimension."):
        po.sample_farthest_points(x, lengths=torch.tensor([5]))
    with pytest.raises(ValueError, match="A value in lengths was too large."):
        po.sample_farthest_points(x, lengths=torch.tensor([5, 6]))
    with pytest.raises(ValueError, match="K and points must have the same batch dimension"):
        po.sample_farthest_points(x, K=[1, 2, 3])
    with pytest.raises(ValueError, match="pts1 and pts2 must have the same batch dimension."):
        po.ball_query(x, torch.zeros(3, 5, 3))
    with pytest.raises(ValueError, match="pts1 and pts2 must have the same point dimension."):
        po.ball_query(x, torch.zeros(2, 5, 2))
    with pytest.raises(ValueError, match="points and idx must have the same batch dimension"):
        po.masked_gather(x, torch.zeros(3, 2, dtype=torch.int64))
    with pytest.raises(ValueError, match="idx format is not supported"):
        po.masked_gather(x, torch.zeros(2, dtype=torch.int64))
    # K = 0 returns (N, 0) without a launch; a negative K raises the reference's size error
    pts, idx = po.sample_farthest_points(x, K=0)
    assert idx.shape == (2, 0) and pts.shape == (2, 0, 3)
    with pytest.raises(RuntimeError, match="negative dimension"):
        po.sample_farthest_points(x, K=-1)


def test_other_d_raises_cpu():
    from pytorch3d_b200 import point_ops as po
    with pytest.raises(ValueError, match="D = 3"):
        po.sample_farthest_points(torch.zeros(2, 5, 2))
    with pytest.raises(ValueError, match="D = 3"):
        po.ball_query(torch.zeros(2, 5, 4), torch.zeros(2, 5, 4))


def test_masked_gather_cpu():
    from pytorch3d_b200 import point_ops as po
    pts = torch.arange(2 * 4 * 3, dtype=torch.float32).view(2, 4, 3)
    idx = torch.tensor([[3, -1], [0, 2]])
    assert po.masked_gather(pts, idx).tolist() == [[[9, 10, 11], [0, 0, 0]], [[12, 13, 14], [18, 19, 20]]]
    idx3 = torch.tensor([[[1, -1]], [[-1, 3]]])
    assert po.masked_gather(pts, idx3).tolist() == [[[[3, 4, 5], [0, 0, 0]]], [[[0, 0, 0], [21, 22, 23]]]]


def _fake_ops_modules(monkeypatch):
    m = types.ModuleType("pytorch3d")
    m.__path__ = []
    monkeypatch.setitem(sys.modules, "pytorch3d", m)
    package = types.ModuleType("pytorch3d.ops")
    package.__path__ = []
    fps_mod = types.ModuleType("pytorch3d.ops.sample_farthest_points")
    ball_mod = types.ModuleType("pytorch3d.ops.ball_query")

    def sample_farthest_points(points, lengths=None, K=50, random_start_point=False):
        return ("ref", K)

    def ball_query(p1, p2, lengths1=None, lengths2=None, K=500, radius=0.2, return_nn=True,
                   skip_points_outside_cube=False):
        return ("ref", K, radius)

    fps_mod.sample_farthest_points = package.sample_farthest_points = sample_farthest_points
    ball_mod.ball_query = package.ball_query = ball_query
    for mod in (package, fps_mod, ball_mod):
        monkeypatch.setitem(sys.modules, mod.__name__, mod)
    return package, fps_mod, ball_mod, sample_farthest_points, ball_query


def test_install_point_ops_routing_and_uninstall_cpu(monkeypatch):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import point_ops as ours
    package, fps_mod, ball_mod, fps_orig, ball_orig = _fake_ops_modules(monkeypatch)
    monkeypatch.setattr(ours, "sample_farthest_points", lambda *a: ("b200",) + a[2:3])
    monkeypatch.setattr(ours, "ball_query", lambda *a: ("b200",) + a[4:6])
    assert inst.install_point_ops() == ["pytorch3d.ops", "pytorch3d.ops.sample_farthest_points",
                                        "pytorch3d.ops.ball_query"]
    x = torch.zeros(2, 4, 3)
    for owner in (package, fps_mod):
        assert owner.sample_farthest_points(x, K=3)[0] == "ref"                       # CPU
        assert owner.sample_farthest_points(x.double().to(DEV) if torch.cuda.is_available() else x.double(),
                                            K=3)[0] == "ref"                          # float64
        assert owner.sample_farthest_points(torch.zeros(2, 4, 2), K=3)[0] == "ref"    # D != 3
    for owner in (package, ball_mod):
        assert owner.ball_query(x, x, K=3)[0] == "ref"
        assert owner.ball_query(torch.zeros(2, 4, 5), torch.zeros(2, 4, 5))[0] == "ref"
    assert not inst._fps_fused(x, None, 3) and not inst._ball_fused(x, x, None, None, 3)
    if torch.cuda.is_available():
        xc = x.to(DEV)
        for owner in (package, fps_mod):
            assert owner.sample_farthest_points(xc, K=3) == ("b200", 3)
            assert owner.sample_farthest_points(xc, lengths=torch.tensor([4, 4]), K=3)[0] == "ref"  # CPU lengths
        for owner in (package, ball_mod):
            assert owner.ball_query(xc, xc, K=3, radius=0.5) == ("b200", 3, 0.5)
            assert owner.ball_query(xc, x, K=3)[0] == "ref"                           # mixed devices
            assert owner.ball_query(xc, xc, K=3.0)[0] == "ref"                        # K not an integer
            assert owner.ball_query(xc, xc, K=1 << 30)[0] == "ref"                    # over the size limit
    inst.install_point_ops()  # idempotent
    inst.uninstall()
    assert package.sample_farthest_points is fps_orig and fps_mod.sample_farthest_points is fps_orig
    assert package.ball_query is ball_orig and ball_mod.ball_query is ball_orig
    assert not any(k[1] in ("sample_farthest_points", "ball_query") for k in inst._saved_blend)


# ---- GPU ---------------------------------------------------------------------------------------------------------

def _ref_cuda():
    from oracle import build_ref_point_ops
    m = build_ref_point_ops.load(cuda=True)
    if m is None:
        pytest.skip("oracle/_ref/ref_point_ops_cuda.so not built (the reference sources were absent at build time)")
    return m


def _ref_knn_cuda():
    from oracle import build_ref_knn
    m = build_ref_knn.load(cuda=True)
    if m is None:
        pytest.skip("oracle/_ref/ref_knn_cuda.so not built (the reference sources were absent at build time)")
    return m


def _fps_inputs(points, lengths=None, K=None, start=None):
    N, P = points.shape[:2]
    lengths = torch.full((N,), P, dtype=torch.int64) if lengths is None else torch.as_tensor(lengths)
    K = torch.as_tensor(K, dtype=torch.int64)
    start = torch.zeros(N, dtype=torch.int64) if start is None else torch.as_tensor(start, dtype=torch.int64)
    return [t.to(DEV) for t in (points.float(), lengths, K, start)]


def _check_fps(ref, points, lengths=None, K=None, start=None, clusters=(0,)):
    from pytorch3d_b200 import _C
    pts, l, k, s = _fps_inputs(points, lengths, K, start)
    max_K = int(k.max())
    want = ref.sample_farthest_points(pts, l, k, s, max_K).cpu()
    for c in clusters:
        got = _C.sample_farthest_points(pts, l, k, s, max_K, c).cpu()
        assert torch.equal(got, want), "cluster size %d differs from the reference kernel" % c


@pytest.mark.gpu
def test_fps_matches_reference_kernel(built_lib):
    ref = _ref_cuda()
    g = torch.Generator().manual_seed(1)
    all_sizes = tuple(range(0, 17))
    _check_fps(ref, torch.rand(4, 3000, 3, generator=g), K=[100, 100, 100, 100], clusters=all_sizes)
    _check_fps(ref, torch.rand(5, 2000, 3, generator=g), lengths=[2000, 1500, 9, 1, 0], K=[300, 0, 20, 5, 3],
               clusters=(0, 1, 3, 16))
    grid = torch.stack(torch.meshgrid(*[torch.arange(12.0)] * 3, indexing="ij"), -1).reshape(1, -1, 3)
    _check_fps(ref, grid.repeat(2, 1, 1), K=[600, 600], start=[0, 777], clusters=(0, 1, 2, 5, 16))
    dup = torch.randint(-2, 3, (2, 40, 3), generator=g).float().repeat(1, 50, 1)
    _check_fps(ref, dup, K=[200, 200], clusters=(0, 1, 7))
    big = torch.rand(2, 1500, 3, generator=g) * 2e6 - 1e6  # squared distances above the 1e10 cap tie there
    _check_fps(ref, big, K=[64, 64], clusters=(0, 1, 4))
    nf = torch.randint(-5, 6, (2, 700, 3), generator=g).float()
    nf[0, 10, 0], nf[0, 20, 1], nf[1, 5, 2], nf[1, 600, 0] = float("nan"), float("inf"), float("-inf"), float("nan")
    _check_fps(ref, nf, K=[30, 30], clusters=(0, 1, 2))
    _check_fps(ref, torch.rand(256, 1024, 3, generator=g), K=[128] * 256)
    _check_fps(ref, torch.rand(1, 1 << 17, 3, generator=g), K=[256], clusters=(0, 16))
    # one cloud beyond the on-chip capacity of a 16-CTA cluster: the L2 tier
    _check_fps(ref, torch.rand(1, 1_000_000, 3, generator=g), K=[48], clusters=(0, 2))


@pytest.mark.gpu
def test_fps_launch_policy_boundaries(built_lib):
    """Cloud sizes +-1 around the register tier of one CTA (4096 points), around the policy's steps of 8192 points per
    CTA up to 16 CTAs, batch sizes where the SMs per cloud change the cluster size, and the shared-memory and L2
    tiers."""
    ref = _ref_cuda()
    g = torch.Generator().manual_seed(2)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for P in (4095, 4096, 4097, 8191, 8192, 8193, 16383, 16384, 16385, 65535, 65536, 65537, 131071, 131072, 131073):
        _check_fps(ref, torch.rand(1, P, 3, generator=g), K=[40])
    # batch sizes where the SMs per cloud (SMs // N) change the cluster size: 2 -> 1 at 9000 points, 5 -> 4 at 40000
    for N, P in ((sms // 2, 9000), (sms // 2 + 1, 9000), (sms // 5, 40000), (sms // 5 + 1, 40000)):
        _check_fps(ref, torch.rand(N, P, 3, generator=g), K=[17] * N)
    # the shared-memory tier of one CTA (4096 points in registers, then up to the opt-in shared memory) and of a
    # 16-CTA cluster, and the L2 tier beyond both
    # fps_kernel's static shared memory is 2 x 9 slots of 24 bytes; 1 KB more is kept free
    smem = (torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 432 - 1024) // 16
    for P in (4096 + smem - 1, 4096 + smem, 4096 + smem + 1, 3 * (4096 + smem)):
        _check_fps(ref, torch.rand(1, P, 3, generator=g), K=[40], clusters=(1,))
    for P in (16 * (4096 + smem) - 1, 16 * (4096 + smem), 16 * (4096 + smem) + 1):
        _check_fps(ref, torch.rand(1, P, 3, generator=g), K=[40], clusters=(0, 16))


@pytest.mark.gpu
def test_fps_small_clouds_against_restatement(built_lib):
    """P < 8, where the reference launches too few CTAs: the correctly launched result."""
    from pytorch3d_b200 import _C
    g = torch.Generator().manual_seed(3)
    for P in range(1, 8):
        pts = torch.randint(-3, 4, (5, P, 3), generator=g).float()
        lengths, K = [P, max(P - 1, 0), 1, 0, P], [P + 1, 3, 2, 2, 0]
        got = _C.sample_farthest_points(*_fps_inputs(pts, lengths, K), max(K)).cpu().numpy()
        np.testing.assert_array_equal(got, fps_restated(pts.numpy(), lengths, K, [0] * 5, max(K)))
    # out-of-range starts and empty clouds, as documented
    pts = torch.rand(3, 50, 3, generator=g)
    got = _C.sample_farthest_points(*_fps_inputs(pts, [50, 50, 0], [4, 4, 4], [50, -3, 9]), 4).cpu()
    assert got.tolist() == [[-1] * 4, [-1] * 4, [9, -1, -1, -1]]
    # max_K below some K[n]: read as max_K
    got = _C.sample_farthest_points(*_fps_inputs(pts, None, [10, 2, 3]), 3).cpu().numpy()
    np.testing.assert_array_equal(got, fps_restated(pts.numpy(), None, [10, 2, 3], [0] * 3, 3))


@pytest.mark.gpu
def test_fps_random_start_matches_reference(built_lib):
    from pytorch3d_b200 import point_ops as po
    ref = _ref_cuda()
    g = torch.Generator().manual_seed(4)
    pts = torch.rand(4, 900, 3, generator=g).to(DEV)
    lengths = torch.tensor([900, 500, 33, 2], device=DEV)
    for lens in (None, lengths):
        torch.manual_seed(11)
        sel, idx = po.sample_farthest_points(pts, lens, K=50, random_start_point=True)
        torch.manual_seed(11)
        if lens is None:
            start = torch.randint(high=900, size=(4,), device=DEV)
            L = torch.full((4,), 900, dtype=torch.int64, device=DEV)
        else:
            start = (lens * torch.rand(lens.size(), device=DEV)).to(torch.int64)
            L = lens
        want = ref.sample_farthest_points(pts, L, torch.full((4,), 50, dtype=torch.int64, device=DEV), start, 50)
        assert torch.equal(idx, want)
        assert torch.equal(sel, po.masked_gather(pts, want))


def _ball_ref(ref, p1, p2, l1, l2, K, radius, skip):
    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    l1 = torch.full((N,), P1, dtype=torch.int64, device=DEV) if l1 is None else l1
    l2 = torch.full((N,), P2, dtype=torch.int64, device=DEV) if l2 is None else l2
    return ref.ball_query(p1, p2, l1, l2, K, radius, skip)


def _ball_cases_gpu():
    g = torch.Generator().manual_seed(6)
    u1, u2 = torch.rand(3, 700, 3, generator=g), torch.rand(3, 1100, 3, generator=g)
    grid = torch.stack(torch.meshgrid(*[torch.arange(-3.0, 4.0)] * 3, indexing="ij"), -1).reshape(1, -1, 3)
    nf1, nf2 = torch.randint(-2, 3, (2, 300, 3), generator=g).float(), torch.randint(-2, 3, (2, 600, 3), generator=g).float()
    nf1[0, 3, 0], nf1[1, 7, 2], nf2[0, 5, 1], nf2[1, 9, 0] = float("nan"), float("inf"), float("-inf"), float("nan")
    rag = [700, 255, 0]
    cases = {
        "uniform_k1": (u1, u2, None, None, 1, 0.2, False), "uniform_k32": (u1, u2, None, None, 32, 0.2, False),
        "uniform_k500": (u1, u2, None, None, 500, 0.5, False), "k_above_p2": (u1, u2[:, :300], None, None, 400, 2.0, False),
        "ragged": (u1, u2, torch.tensor(rag), torch.tensor([1100, 0, 513]), 32, 0.3, False),
        "grid_on_radius": (grid, grid, None, None, 40, 2.0, False), "grid_skip": (grid, grid, None, None, 40, 2.0, True),
        "all_hit": (u1, u2, None, None, 1100, 10.0, True), "no_hit": (u1, u2, None, None, 16, 0.0, False),
        "negative": (u1, u2, None, None, 16, -0.2, False), "negative_skip": (u1, u2, None, None, 16, -0.2, True),
        "nonfinite": (nf1, nf2, None, None, 64, 1.5, False), "nonfinite_skip": (nf1, nf2, None, None, 64, 1.5, True),
    }
    for P2 in (511, 512, 513, 1024, 1025):  # tile boundaries of the target stream; 255 / 257 queries per CTA
        cases["tiles_%d" % P2] = (torch.rand(2, 257, 3, generator=g), torch.rand(2, P2, 3, generator=g), None,
                                  None, 600, 0.9, False)
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(_ball_cases_gpu()))
def test_ball_query_matches_reference_kernel(built_lib, case):
    from pytorch3d_b200 import _C, point_ops as po
    ref = _ref_cuda()
    p1, p2, l1, l2, K, radius, skip = _ball_cases_gpu()[case]
    p1, p2 = p1.to(DEV), p2.to(DEV)
    l1, l2 = (None if t is None else t.to(DEV) for t in (l1, l2))
    want_idx, want_d = _ball_ref(ref, p1, p2, l1, l2, K, radius, skip)
    idx, dists, nn = _C.ball_query_forward(p1, p2, l1, l2, K, radius, skip, True)
    assert torch.equal(idx, want_idx)
    assert torch.equal(dists.view(torch.int32), want_d.view(torch.int32))
    assert torch.equal(nn.view(torch.int32), po.masked_gather(p2, idx).view(torch.int32))
    idx2, d2 = _C.ball_query(p1, p2, l1, l2, K, radius, skip)
    assert torch.equal(idx2, idx) and torch.equal(d2, dists)


def _grad_case(seed=7, N=2, P1=300, P2=500, K=24, radius=0.25):
    g = torch.Generator().manual_seed(seed)
    p1, p2 = torch.rand(N, P1, 3, generator=g), torch.rand(N, P2, 3, generator=g)
    gd, gnn = torch.randn(N, P1, K, generator=g), torch.randn(N, P1, K, 3, generator=g)
    return p1, p2, gd, gnn, K, radius


@pytest.mark.gpu
@pytest.mark.parametrize("upstream", ["dists", "nn", "both"])
def test_ball_query_gradients(built_lib, upstream):
    from pytorch3d_b200 import point_ops as po
    p1, p2, gd, gnn, K, radius = _grad_case()
    l1, l2 = torch.tensor([300, 211]), torch.tensor([500, 377])
    a, b = p1.to(DEV).requires_grad_(), p2.to(DEV).requires_grad_()
    out = po.ball_query(a, b, l1.to(DEV), l2.to(DEV), K=K, radius=radius)
    loss = 0
    if upstream in ("dists", "both"):
        loss = loss + (out.dists * gd.to(DEV)).sum()
    if upstream in ("nn", "both"):
        loss = loss + (out.knn * gnn.to(DEV)).sum()
    loss.backward()
    idx = out.idx.cpu().numpy()
    assert (idx >= 0).sum() > 1000
    want1, want2 = ball_grad_restated(p1.numpy(), p2.numpy(), idx, gd.numpy() if upstream != "nn" else None,
                                      gnn.numpy() if upstream != "dists" else None)
    # per element: the float32 sums of at most K + (i, k) terms against float64
    for got, want in ((a.grad, want1), (b.grad, want2)):
        got = got.cpu().double().numpy()
        scale = np.abs(want).max()
        np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-6 * scale)
    # against the reference's chain: its CUDA ball query, knn_points_backward (float atomics) and torch's gather
    ref, knn = _ref_cuda(), _ref_knn_cuda()
    ridx, rd = ref.ball_query(p1.to(DEV), p2.to(DEV), l1.to(DEV), l2.to(DEV), K, radius, False)
    assert torch.equal(ridx, out.idx)
    r1 = torch.zeros_like(a)
    r2 = torch.zeros_like(b)
    if upstream != "nn":
        r1, r2 = knn.knn_points_backward(p1.to(DEV), p2.to(DEV), l1.to(DEV), l2.to(DEV), ridx, 2, gd.to(DEV))
    if upstream != "dists":
        bb = p2.to(DEV).requires_grad_()
        (po.masked_gather(bb, ridx) * gnn.to(DEV)).sum().backward()
        r2 = r2 + bb.grad
    torch.testing.assert_close(a.grad, r1, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(b.grad, r2, rtol=1e-5, atol=1e-5)


@pytest.mark.gpu
def test_ball_query_backward_chunks(built_lib):
    """More sorted rows than one chunk of the grad_p2 pass: the chunks continue each other's sums."""
    from pytorch3d_b200 import _C
    g = torch.Generator().manual_seed(8)
    p1, p2 = torch.rand(2, 3000, 3, generator=g), torch.rand(2, 2000, 3, generator=g)
    K = 200  # 2 * 3000 * 200 = 1.2 M rows
    idx, _, _ = _C.ball_query_forward(p1.to(DEV), p2.to(DEV), None, None, K, 0.3, False, False)
    gd, gnn = torch.randn(2, 3000, K, generator=g), torch.randn(2, 3000, K, 3, generator=g)
    g1, g2 = _C.ball_query_backward(p1.to(DEV), p2.to(DEV), None, None, idx, gd.to(DEV), gnn.to(DEV))
    w1, w2 = ball_grad_restated(p1.numpy(), p2.numpy(), idx.cpu().numpy(), gd.numpy(), gnn.numpy())
    for got, want in ((g1, w1), (g2, w2)):
        np.testing.assert_allclose(got.cpu().double().numpy(), want, rtol=1e-4, atol=1e-4)


@pytest.mark.gpu
def test_determinism(built_lib):
    from pytorch3d_b200 import point_ops as po
    p1, p2, gd, gnn, K, radius = _grad_case(seed=9, K=64, radius=0.4)
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            a, b = p1.to(DEV).requires_grad_(), p2.to(DEV).requires_grad_()
            sel, fidx = po.sample_farthest_points(b, K=64)
            out = po.ball_query(a, b, K=K, radius=radius)
            ((out.dists * gd.to(DEV)).sum() + (out.knn * gnn.to(DEV)).sum() + sel.square().sum()).backward()
            runs.append([t.detach().cpu() for t in (fidx, out.idx, out.dists, out.knn, a.grad, b.grad)])
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y in zip(*runs):
        assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x,
                           y.view(torch.uint8) if y.is_floating_point() else y)


def _count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return len([w for w in rec if "synchroniz" in str(w.message)])


@pytest.mark.gpu
def test_host_synchronisations(built_lib):
    from pytorch3d_b200 import point_ops as po
    p1, p2, gd, gnn, K, radius = _grad_case(seed=10)
    a, b = p1.to(DEV).requires_grad_(), p2.to(DEV).requires_grad_()
    out = {}
    assert _count_syncs(lambda: out.setdefault("q", po.ball_query(a, b, K=K, radius=radius))) == 0
    q = out["q"]
    loss = (q.dists * gd.to(DEV)).sum() + (q.knn * gnn.to(DEV)).sum()
    assert _count_syncs(lambda: loss.backward()) == 0
    x = p2.to(DEV)
    assert _count_syncs(lambda: po.sample_farthest_points(x, K=16)) == 0
    assert _count_syncs(lambda: po.sample_farthest_points(x, K=[16, 9])) == 0
    lengths = torch.tensor([500, 300], device=DEV)
    Kt = torch.tensor([16, 9], device=DEV)
    assert _count_syncs(lambda: po.sample_farthest_points(x, lengths, K=16)) <= 1
    assert _count_syncs(lambda: po.sample_farthest_points(x, K=Kt)) <= 1
    assert _count_syncs(lambda: po.sample_farthest_points(x, lengths, K=Kt)) <= 1


@pytest.mark.gpu
def test_ball_query_backward_peak_memory(built_lib):
    """At K = 500 the backward with nn stays below the (N, P2, K, 3) float32 buffer of the reference's gather: what
    the op itself allocates, given the upstream gradients."""
    from pytorch3d_b200 import point_ops as po
    g = torch.Generator().manual_seed(12)
    N, P, K = 4, 4096, 500
    a = torch.rand(N, P, 3, generator=g).to(DEV).requires_grad_()
    b = torch.rand(N, P, 3, generator=g).to(DEV).requires_grad_()
    out = po.ball_query(a, b, K=K, radius=0.2)
    gd, gnn = torch.randn_like(out.dists), torch.randn_like(out.knn)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.autograd.backward([out.dists, out.knn], [gd, gnn])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < N * P * K * 3 * 4, (peak, N * P * K * 3 * 4)


@pytest.mark.gpu
def test_argument_checks(built_lib):
    """The ctypes ops refuse a wrong dtype or shape with RuntimeError naming the argument, before any launch."""
    from pytorch3d_b200 import _C, _lib
    p1, p2 = torch.rand(2, 10, 3, device=DEV), torch.rand(2, 12, 3, device=DEV)
    L = torch.tensor([10, 10], device=DEV)
    K = torch.tensor([3, 3], device=DEV)
    s = torch.zeros(2, dtype=torch.int64, device=DEV)
    idx, _, _ = _C.ball_query_forward(p1, p2, None, None, 4, 0.5, False, False)
    g = torch.zeros(2, 10, 4, device=DEV)
    torch.cuda.synchronize()
    before = _lib.load().b200r_kernel_launch_count()
    bad = [
        (lambda: _C.sample_farthest_points(p1.double(), L, K, s, 3), "points"),
        (lambda: _C.sample_farthest_points(p1[..., :2].contiguous(), L, K, s, 3), "points"),
        (lambda: _C.sample_farthest_points(p1, L.int(), K, s, 3), "lengths"),
        (lambda: _C.sample_farthest_points(p1, L, K.float(), s, 3), "K"),
        (lambda: _C.sample_farthest_points(p1, L, K, s[:1], 3), "start_idxs"),
        (lambda: _C.ball_query_forward(p1.half(), p2, None, None, 4, 0.5, False, False), "p1"),
        (lambda: _C.ball_query_forward(p1, p2[:1], None, None, 4, 0.5, False, False), "p2"),
        (lambda: _C.ball_query_forward(p1, p2, L.int(), None, 4, 0.5, False, False), "lengths1"),
        (lambda: _C.ball_query_forward(p1, p2, None, L[:1], 4, 0.5, False, False), "lengths2"),
        (lambda: _C.ball_query_backward(p1, p2, None, None, idx.int(), g, None), "idx"),
        (lambda: _C.ball_query_backward(p1, p2, None, None, idx, g[..., :3], None), "grad_dists"),
        (lambda: _C.ball_query_backward(p1, p2, None, None, idx, None, torch.zeros(2, 10, 4, 2, device=DEV)),
         "grad_nn"),
        (lambda: _C.ball_query_backward(p1, p2[:, :, :2], None, None, idx, g, None), "p2"),
    ]
    for fn, name in bad:
        with pytest.raises(RuntimeError, match=name):
            fn()
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.ball_query_forward(p1.cpu(), p2, None, None, 4, 0.5, False, False)
    assert _lib.load().b200r_kernel_launch_count() == before


@pytest.mark.gpu
def test_pointnet2_set_abstraction_step(built_lib):
    """FPS, ball query, grouped relative coordinates, a small shared MLP pooled over each ball, backward."""
    from pytorch3d_b200 import point_ops as po
    torch.manual_seed(13)
    N, P, S, K = 4, 2048, 256, 32
    xyz = torch.rand(N, P, 3, device=DEV, requires_grad=True)
    mlp = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.ReLU(), torch.nn.Linear(32, 64)).to(DEV)
    centres, _ = po.sample_farthest_points(xyz, K=S)
    out = po.ball_query(centres, xyz, K=K, radius=0.15)
    valid = (out.idx >= 0)
    grouped = (out.knn - centres[:, :, None, :]) * valid[..., None]
    feats = (mlp(grouped) * valid[..., None]).sum(dim=2)
    loss = feats.square().mean() + out.dists.mean()
    loss.backward()
    assert torch.isfinite(loss)
    assert torch.isfinite(xyz.grad).all()
    assert valid.sum() > N * S  # more than the centres themselves
    grouped_pts = torch.zeros(N, P, device=DEV).scatter_add_(1, out.idx.clamp(min=0).view(N, -1),
                                                            valid.view(N, -1).float()) > 0
    assert (xyz.grad.abs().sum(-1)[grouped_pts] > 0).all()
