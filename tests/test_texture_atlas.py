"""Texture atlas sampling (DESIGN.md section 15): the fused `sample_textures_atlas` / `sample_textures` against a torch
restatement of the reference's TexturesAtlas.sample_textures (pytorch3d/renderer/mesh/textures.py), and
`install_texture_atlas()`.

The stored outputs of the reference (tests/golden/reference_golden_atlas.npz, tests/golden/make_atlas_golden.py) pin
the restatement below to the reference: its own textures module runs on the CPU."""
import sys
import types

import numpy as np
import pytest
import torch

from helpers import reference

# ------------------------------------------------------------------------------------------------ scenes
# (R, C, how the texture is built): R in {1, 2, 3, 4, 8}, C in {1, 3, 4, 7}, list- and padded-built atlases
ATLAS_CASES = [(1, 3, "list"), (2, 1, "padded"), (3, 4, "list"), (4, 3, "padded"), (4, 7, "list"), (8, 3, "list"),
               (8, 4, "padded"), (1, 7, "padded"), (3, 1, "padded"), (2, 3, "list")]
SCENE = (2, 5, 7, 3)  # N, H, W, K: non-square
FACES = (5, 3)  # faces of the two meshes
FIELDS = ("texels", "grad_atlas")


def atlas_case(args):
    R, C, build = args
    return "atlas/R%d-C%d-%s" % (R, C, build)


def special_barys(R):
    """(b0, b1, b2) rows: corners, cell boundaries (b·R an integer), the diagonal test's equality, b0 > 1 (the clamp)
    and b0 in [-1, 0) (the negative index wraps).  Every row indexes the atlas (none is out of range)."""
    rows = [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (0.5, 0.5, 0.0)]
    for k in range(R + 1):
        for j in range(R + 1 - k):
            rows.append((k / R, j / R, 1.0 - (k + j) / R))  # cell boundaries
    for k in range(R):
        rows.append(((k + 0.5) / R, (R - 1 - k + 0.5) / R, 0.0))  # (b0 + b1)·R − (w0 + w1) == 1 when R is dyadic
        rows.append(((k + 0.25) / R, (0.75) / R, 0.0))
    rows += [(1.25, 0.1, -0.35), (1.5, 0.0, -0.5), (1.0625, 0.25, -0.3125)]  # clamp to R − 1, then flipped
    rows += [(-0.5, 0.25, 1.25), (-1.0, 0.0, 2.0), (-0.125, 0.5, 0.625), (0.25, -0.75, 1.5)]  # wrap, not flipped
    return torch.tensor(rows, dtype=torch.float32)


def atlas_scene(N, H, W, K, R, C, faces=None, seed=0, frac_background=0.3, device="cpu"):
    """A dict: the per-mesh atlases (a list of (F_i, R, R, C), different face counts) with negative values in cell (0, 0)
    of the last face; pix_to_face into the packed faces of each image's own mesh with about `frac_background`
    background slots; barycentrics, with every row of `special_barys` on a foreground slot where space allows; an
    upstream gradient that is nonzero everywhere, background slots included."""
    faces = faces or FACES[:N] + (FACES[-1],) * max(0, N - len(FACES))
    g = torch.Generator().manual_seed(seed + 1000 * K + 31 * H + W + 7 * R + C)
    atlases = [torch.randn(f, R, R, C, generator=g) for f in faces]
    atlases[-1][-1, 0, 0] = -atlases[-1][-1, 0, 0].abs() - 0.5
    first = torch.tensor([0] + list(faces[:-1])).cumsum(0)
    num = torch.tensor(faces)
    img = torch.arange(N).view(N, 1, 1, 1)
    p2f = (torch.rand(N, H, W, K, generator=g) * num[img]).long() + first[img]
    p2f[torch.rand(N, H, W, K, generator=g) < frac_background] = -1
    bary = torch.rand(N, H, W, K, 3, generator=g) + 0.02
    bary = bary / bary.sum(-1, keepdim=True)
    sp = special_barys(R)
    order = torch.randperm(N * H * W * K, generator=g)
    fg = order[p2f.view(-1)[order] >= 0][:len(sp)]  # every special row on a foreground slot, where space allows
    bary.view(-1, 3)[fg] = sp[:len(fg)]
    s = {"atlases": atlases, "pix_to_face": p2f, "bary": bary, "grad_texels": torch.randn(N, H, W, K, C, generator=g)}
    return {k: ([a.to(device) for a in v] if isinstance(v, list) else v.to(device)) for k, v in s.items()}


def case_scene(args, device="cpu"):
    R, C, _ = args
    return atlas_scene(*SCENE, R, C, device=device)


def out_of_range_scene(device="cpu"):
    """R = 4 with one slot at b = (-0.5, 1.5, 0): w = (-2, 3), flipped to (5, 0), past the end of the patch."""
    s = atlas_scene(1, 2, 3, 2, 4, 3, faces=(4,), seed=5, frac_background=0.0)
    s["bary"][0, 1, 2, 1] = torch.tensor([-0.5, 1.5, 0.0])
    return {k: ([a.to(device) for a in v] if isinstance(v, list) else v.to(device)) for k, v in s.items()}


# ------------------------------------------------------------------------------------------------ restatement
def chain_sample(fragments, atlas_packed):
    """TexturesAtlas.sample_textures in the reference's operations, on the packed atlas (F, R, R, C)."""
    p2f, bary = fragments.pix_to_face, fragments.bary_coords
    R = atlas_packed.shape[1]
    background = (p2f < 0)[..., None]
    b01 = torch.where(background, torch.zeros_like(bary[..., :2]), bary[..., :2])
    w = (b01 * R).to(torch.int64).clamp(max=R - 1)
    below = (b01.sum(dim=-1) * R - w.float().sum(dim=-1)) <= 1.0
    wx, wy = w.unbind(-1)
    wx = torch.where(below, wx, R - 1 - wx)
    wy = torch.where(below, wy, R - 1 - wy)
    return atlas_packed[p2f, wy, wx] * (p2f >= 0)[..., None].float()


def assert_cells_in_range(fragments, atlas_packed):
    """Checks on the CPU that the chain can index every slot's cell: on CUDA its gather would fail a device-side
    assertion instead of raising."""
    F, R = int(atlas_packed.shape[0]), int(atlas_packed.shape[1])
    frags = types.SimpleNamespace(pix_to_face=fragments.pix_to_face.detach().cpu(),
                                  bary_coords=fragments.bary_coords.detach().cpu())
    cells = torch.arange(F * R * R, dtype=torch.float32).view(F, R, R, 1)
    chain_sample(frags, cells)  # IndexError here if any cell is out of range


def fused_sample(fragments, atlas_packed):
    from pytorch3d_b200.texture_atlas import sample_textures_atlas
    return sample_textures_atlas(fragments, atlas_packed)


def leaf_atlas(s, build):
    """(leaf the gradient lands on, packed atlas) built as a list- or padded-built TexturesAtlas packs it."""
    if build == "list":
        leaves = [a.clone().requires_grad_(True) for a in s["atlases"]]
        return leaves, torch.cat(leaves)
    F = max(a.shape[0] for a in s["atlases"])
    padded = torch.zeros((len(s["atlases"]), F) + tuple(s["atlases"][0].shape[1:]), device=s["bary"].device)
    for i, a in enumerate(s["atlases"]):
        padded[i, :a.shape[0]] = a
    padded.requires_grad_(True)
    return padded, torch.cat([padded[i, :a.shape[0]] for i, a in enumerate(s["atlases"])])


def with_grads(fn, s, build="list"):
    """[(name, tensor)]: the texels and the gradient of the atlas the texture was built from (the list's gradients
    concatenated, or the padded tensor's) under the scene's upstream gradient; asserts the barycentrics get none."""
    leaf, packed = leaf_atlas(s, build)
    bary = s["bary"].clone().requires_grad_(True)
    frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=bary)
    if fn is chain_sample and bary.is_cuda:
        assert_cells_in_range(frags, packed)
    texels = fn(frags, packed)
    (texels * s["grad_texels"]).sum().backward()
    assert bary.grad is None
    grad = torch.cat([t.grad for t in leaf]) if build == "list" else leaf.grad
    return list(zip(FIELDS, [texels.detach(), grad]))


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("args", ATLAS_CASES, ids=[atlas_case(a)[6:] for a in ATLAS_CASES])
def test_atlas_chain_equals_reference_cpu(args):
    got = with_grads(chain_sample, case_scene(args), args[2])
    for name, t in got:
        err = reference(atlas_case(args) + "/" + name)[0].equals(t)
        assert err is None, "%s %s: torch restatement vs the reference (CPU): %s" % (atlas_case(args), name, err)


def test_scenes_cover_the_special_cases():
    for R, C, _ in ATLAS_CASES:
        s = atlas_scene(*SCENE, R, C)
        b, p2f = s["bary"], s["pix_to_face"]
        fg = p2f >= 0
        assert 0.2 < float((~fg).float().mean()) < 0.4
        assert (b[fg][:, 0] > 1).any() and ((b[fg][:, 0] < 0) & (b[fg][:, 0] >= -1)).any()
        bR = b[fg][:, :2] * R
        assert (bR == bR.trunc()).all(dim=-1).any()  # on cell boundaries
        w = bR.to(torch.int64).clamp(max=R - 1)
        if R in (1, 2, 4, 8):
            assert ((b[fg][:, :2].sum(-1) * R - w.float().sum(-1)) == 1.0).any()  # the diagonal's equality
        assert float(s["atlases"][-1][-1, 0, 0].max()) < 0


def test_out_of_range_raises_in_the_reference_and_the_restatement():
    assert reference("atlas/out_of_range/raises")[0].sample.tolist() == [1]
    s = out_of_range_scene()
    frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=s["bary"])
    with pytest.raises(IndexError):
        chain_sample(frags, torch.cat(s["atlases"]))


def test_key_bits():
    from pytorch3d_b200._C import texture_atlas_key_bits
    assert texture_atlas_key_bits(0, 1) == (1, 4)
    assert texture_atlas_key_bits(1, 1) == (1, 4)  # cells 1: keys 0 and the sentinel 1
    assert texture_atlas_key_bits(2, 1) == (2, 4)
    assert texture_atlas_key_bits(559504, 4) == (24, 4)  # 8,952,064 cells
    assert texture_atlas_key_bits(2 ** 28, 4) == (33, 8)  # 2^32 cells: the sentinel needs bit 32
    assert texture_atlas_key_bits(2 ** 28 - 1, 4) == (32, 4)
    assert texture_atlas_key_bits(2 ** 20 + 1, 64) == (33, 8)


def test_atlas_argument_errors():
    from pytorch3d_b200 import _C
    s = atlas_scene(2, 3, 4, 2, 4, 3)
    p2f, bary, atlas = s["pix_to_face"], s["bary"], torch.cat(s["atlases"])
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.texture_atlas_forward(p2f, bary, atlas)
    with pytest.raises(RuntimeError, match="barycentric_coords must be"):
        _C.texture_atlas_forward(p2f, bary[..., :2], atlas)
    with pytest.raises(RuntimeError, match="atlas must be"):
        _C.texture_atlas_forward(p2f, bary, atlas[:, :, :2])
    with pytest.raises(RuntimeError, match="atlas must be"):
        _C.texture_atlas_forward(p2f, bary, atlas[:, :0, :0])
    with pytest.raises(RuntimeError, match="pix_to_face must have dimensions"):
        _C.texture_atlas_forward(p2f[0], bary, atlas)


class _TexturesAtlas:
    """A stand-in for PyTorch3D's TexturesAtlas (routing looks at the packed atlas only)."""

    def __init__(self, atlas):
        self._atlas = atlas
        self.packed = 0

    def atlas_packed(self):
        self.packed += 1
        return self._atlas


def _fake_atlas_module(monkeypatch):
    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    mod = types.ModuleType("pytorch3d.renderer.mesh.textures")

    class TexturesAtlas(_TexturesAtlas):
        def sample_textures(self, fragments, **kwargs):  # defined on the class itself, as in PyTorch3D
            self.atlas_packed()
            return "ref"

    class TexturesUV:
        def sample_textures(self, fragments, **kwargs):
            return "ref-uv"

    mod.TexturesAtlas, mod.TexturesUV = TexturesAtlas, TexturesUV
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.mesh.textures", mod)
    return TexturesAtlas


def _stand_in(shape, dtype=torch.float32, is_cuda=True, device=None):
    """An object that claims to be a tensor on the GPU (routing looks at device, dtype and shape only)."""
    device = torch.device(device or ("cuda:0" if is_cuda else "cpu"))
    return types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size(shape), dim=lambda: len(shape),
                                 device=device)


def test_install_texture_atlas_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import texture_atlas as ours
    cls = _fake_atlas_module(monkeypatch)
    original = cls.__dict__["sample_textures"]
    routed = []
    monkeypatch.setattr(ours, "sample_textures_atlas", lambda frags, atlas: routed.append(atlas) or "b200")
    assert inst.install_texture_atlas() == ["pytorch3d.renderer.mesh.textures"]
    assert cls.__dict__["sample_textures"] is not original
    frags = types.SimpleNamespace(pix_to_face=_stand_in((2, 4, 5, 3), torch.int64),
                                  bary_coords=_stand_in((2, 4, 5, 3, 3)))
    for R, C in ((1, 3), (4, 3), (8, 7)):
        tex = cls(_stand_in((10, R, R, C)))
        assert tex.sample_textures(frags) == "b200"
        assert tex.packed == 1 and routed[-1] is tex._atlas  # packed once, and that tensor is sampled
    assert len(routed) == 3
    cpu_frags = types.SimpleNamespace(pix_to_face=_stand_in((2, 4, 5, 3), torch.int64, is_cuda=False),
                                      bary_coords=_stand_in((2, 4, 5, 3, 3), is_cuda=False))
    i32_frags = types.SimpleNamespace(pix_to_face=_stand_in((2, 4, 5, 3), torch.int32), bary_coords=frags.bary_coords)
    f64_frags = types.SimpleNamespace(pix_to_face=frags.pix_to_face,
                                      bary_coords=_stand_in((2, 4, 5, 3, 3), torch.float64))
    dev1_frags = types.SimpleNamespace(pix_to_face=frags.pix_to_face,
                                       bary_coords=_stand_in((2, 4, 5, 3, 3), device="cuda:1"))
    atlas = _stand_in((10, 4, 4, 3))
    fallbacks = [
        (cls(_stand_in((2, 0, 0, 3))), frags),  # an empty texture packs to R = 0
        (cls(_stand_in((10, 4, 4, 3), is_cuda=False)), frags),
        (cls(atlas), cpu_frags),
        (cls(_stand_in((10, 4, 4, 3), torch.float64)), frags),
        (cls(atlas), f64_frags),
        (cls(atlas), i32_frags),
        (cls(atlas), dev1_frags),
        (cls(_stand_in((10, 4, 4, 3), device="cuda:1")), frags),
        (cls(_stand_in((10, 4, 4))), frags),
    ]
    for tex, fr in fallbacks:
        assert tex.sample_textures(fr) == "ref"
    assert len(routed) == 3
    inst.uninstall()
    assert cls.__dict__["sample_textures"] is original
    assert inst._saved_methods == {}


def test_install_texture_atlas_leaves_the_other_installs_alone(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    mod_cls = _fake_atlas_module(monkeypatch)
    uv = sys.modules["pytorch3d.renderer.mesh.textures"].TexturesUV
    uv_method = uv.__dict__["sample_textures"]
    inst.install_texture_atlas()
    try:
        assert set(inst._saved_methods) == {("pytorch3d.renderer.mesh.textures", "TexturesAtlas", "sample_textures")}
        assert inst._saved == {} and inst._saved_blend == {}
        assert uv.__dict__["sample_textures"] is uv_method
    finally:
        inst.uninstall()
    assert inst._saved_methods == {} and "sample_textures" in mod_cls.__dict__


def test_drop_in_packs_the_atlas_once(monkeypatch):
    from pytorch3d_b200 import texture_atlas as ours
    seen = []
    monkeypatch.setattr(ours, "sample_textures_atlas", lambda frags, atlas: seen.append((frags, atlas)) or "texels")
    atlas = torch.zeros(3, 2, 2, 3)
    tex = _TexturesAtlas(atlas)
    assert ours.sample_textures(tex, "frags") == "texels"
    assert tex.packed == 1 and seen == [("frags", atlas)]


# ------------------------------------------------------------------------------------------------ GPU tests
DEV = "cuda:0"


def _close(a, b, what):
    """rtol 1e-4 / atol 1e-5 of the largest magnitude."""
    a, b = a.detach().cpu().double().numpy(), b.detach().cpu().double().numpy()
    atol = 1e-5 * float(np.abs(b).max()) + 1e-30
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    ok = np.abs(a - b) <= atol + 1e-4 * np.abs(b)
    assert ok.all(), "%s: %d values differ, max abs diff %g" % (what, int((~ok).sum()), float(np.abs(a - b).max()))


def _contributions(s, build):
    """Per cell of the built atlas: how many slots add a nonzero upstream gradient into it (the chain's own gather)."""
    frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=s["bary"])
    nonzero = (s["grad_texels"] * (s["pix_to_face"] >= 0)[..., None].float() != 0).any(-1, keepdim=True).float()
    cells = torch.cat([a[..., :1] for a in s["atlases"]]).requires_grad_(True)
    (chain_sample(frags, cells) * nonzero).sum().backward()  # counts the slots that add into each cell
    counts = cells.grad[..., 0]
    if build == "list":
        return counts
    F = max(a.shape[0] for a in s["atlases"])
    out = torch.zeros((len(s["atlases"]), F) + tuple(counts.shape[1:]), device=counts.device)
    start = 0
    for i, a in enumerate(s["atlases"]):
        out[i, :a.shape[0]] = counts[start:start + a.shape[0]]
        start += a.shape[0]
    return out


def _compare(s, build, what):
    """Texels bit for bit; the atlas gradient within tolerance, and bit for bit where a cell has at most one
    contribution."""
    got = dict(with_grads(fused_sample, s, build))
    want = dict(with_grads(chain_sample, s, build))
    a, b = got["texels"], want["texels"]
    assert torch.equal(a, b) and torch.equal(torch.signbit(a), torch.signbit(b)), \
        "%s texels: %d differ" % (what, int((a != b).sum()))
    _close(got["grad_atlas"], want["grad_atlas"], what + " grad_atlas")
    single = _contributions(s, build) <= 1
    ga, gb = got["grad_atlas"], want["grad_atlas"]
    assert torch.equal(ga[single], gb[single]), "%s grad_atlas: cells with one contribution differ" % what
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("args", ATLAS_CASES, ids=[atlas_case(a)[6:] for a in ATLAS_CASES])
def test_fused_matches_reference_records(built_lib, args):
    s = case_scene(args, device=DEV)
    got = _compare(s, args[2], atlas_case(args))
    err = reference(atlas_case(args) + "/texels")[0].equals(got["texels"])
    assert err is None, "%s texels vs the reference: %s" % (atlas_case(args), err)
    ref = reference(atlas_case(args) + "/grad_atlas")[0]
    mine = ref.rows_of(got["grad_atlas"])
    assert np.all(np.abs(mine - ref.sample) <= 1e-5 * max(ref.absmax, 1e-30) + 1e-4 * np.abs(ref.sample))


@pytest.mark.gpu
@pytest.mark.parametrize("args", ATLAS_CASES[:6], ids=[atlas_case(a)[6:] for a in ATLAS_CASES[:6]])
@pytest.mark.parametrize("K", [1, 2, 8, 50, 200])
def test_fused_matches_torch_chain(built_lib, K, args):
    R, C, build = args
    _compare(atlas_scene(2, 6, 11, K, R, C, seed=1, device=DEV), build, "K=%d %s" % (K, atlas_case(args)))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 1, 40, 2), (1, 37, 1, 3), (3, 8, 32, 8), (1, 2, 2, 1)])
def test_fused_matches_torch_chain_on_odd_sizes(built_lib, shape):
    for R, C in ((1, 1), (3, 2), (8, 7)):
        s = atlas_scene(*shape, R, C, seed=3, device=DEV)
        _compare(s, "list", "shape=%s R=%d C=%d" % (shape, R, C))


@pytest.mark.gpu
def test_deterministic_mode_and_no_host_sync(built_lib):
    """Under torch.use_deterministic_algorithms(True) both the fused op and the chain run forward and backward; two
    fused runs are bitwise equal, also with torch's sync-debug mode set to raise on a host synchronisation."""
    s = atlas_scene(4, 64, 64, 8, 4, 3, faces=(300, 200, 500, 100), seed=11, device=DEV)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        chain = dict(with_grads(chain_sample, s))
        first = dict(with_grads(fused_sample, s))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            second = dict(with_grads(fused_sample, s))
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        torch.use_deterministic_algorithms(was)
    for name in FIELDS:
        assert torch.equal(first[name], second[name]), name
    assert torch.equal(first["texels"], chain["texels"])
    _close(first["grad_atlas"], chain["grad_atlas"], "deterministic mode")


@pytest.mark.gpu
def test_worst_case_contention_is_reproducible(built_lib):
    """R = 1 and every slot on one face: one cell sums all of them.  Bitwise reproducible, and within tolerance of a
    float64 sum."""
    N, H, W, K, C = 2, 128, 128, 8, 3
    g = torch.Generator().manual_seed(4)
    s = {"atlases": [torch.randn(3, 1, 1, C, generator=g).to(DEV)],
         "pix_to_face": torch.ones((N, H, W, K), dtype=torch.int64, device=DEV),
         "bary": torch.rand(N, H, W, K, 3, generator=g).to(DEV),
         "grad_texels": torch.randn(N, H, W, K, C, generator=g).to(DEV)}
    first = dict(with_grads(fused_sample, s))["grad_atlas"]
    second = dict(with_grads(fused_sample, s))["grad_atlas"]
    assert torch.equal(first, second)
    exact = s["grad_texels"].double().reshape(-1, C).sum(0)
    assert torch.equal(first[0], torch.zeros_like(first[0])) and torch.equal(first[2], torch.zeros_like(first[2]))
    err = (first[1, 0, 0].double() - exact).abs().max()
    assert float(err) <= 1e-5 * float(s["grad_texels"].abs().sum()) / C, float(err)


@pytest.mark.gpu
def test_infinite_upstream_gradient_on_a_background_slot(built_lib):
    """Background slots read atlas[F-1, 0, 0] times 0: an inf upstream gradient there makes that cell's gradient NaN,
    in the chain and in the fused op; every other cell is unaffected."""
    s = atlas_scene(2, 4, 5, 3, 4, 3, seed=6, device=DEV)
    bg = (s["pix_to_face"] < 0).nonzero()[0].tolist()
    s["grad_texels"][tuple(bg)] = torch.tensor([float("inf"), 1.0, 2.0], device=DEV)
    got = dict(with_grads(fused_sample, s))["grad_atlas"]
    want = dict(with_grads(chain_sample, s))["grad_atlas"]
    assert torch.isnan(got[-1, 0, 0, 0]) and torch.isnan(want[-1, 0, 0, 0])
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    finite = ~torch.isnan(want)
    _close(got[finite], want[finite], "finite cells")


@pytest.mark.gpu
def test_out_of_range_cells_give_zero_on_the_fused_op(built_lib):
    """The reference raises on these slots (IndexError on the CPU, a device-side assert on CUDA); the fused op gives
    texel 0 and no gradient.  Only the fused op runs here."""
    from pytorch3d_b200 import _C
    s = out_of_range_scene(device=DEV)
    atlas = torch.cat(s["atlases"])
    texels = _C.texture_atlas_forward(s["pix_to_face"], s["bary"], atlas)
    assert torch.equal(texels[0, 1, 2, 1], torch.zeros(3, device=DEV))
    g = torch.zeros_like(s["grad_texels"])
    g[0, 1, 2, 1] = 1.0
    grad = _C.texture_atlas_backward(g, s["pix_to_face"], s["bary"], atlas)
    assert int(grad.count_nonzero()) == 0
    # every other slot is what the chain gives with that slot moved into range
    s_cpu = out_of_range_scene()
    s_cpu["bary"][0, 1, 2, 1] = torch.tensor([0.2, 0.3, 0.5])
    frags = types.SimpleNamespace(pix_to_face=s_cpu["pix_to_face"], bary_coords=s_cpu["bary"])
    want = chain_sample(frags, torch.cat(s_cpu["atlases"])).to(DEV)
    keep = torch.ones(texels.shape[:4], dtype=torch.bool, device=DEV)
    keep[0, 1, 2, 1] = False
    assert torch.equal(texels[keep], want[keep])


@pytest.mark.gpu
def test_atlas_past_2_to_the_32_cells(built_lib):
    """An atlas of 2^20 + 1 faces at R = 64, C = 1: 4.29e9 floats (17.2 GB), whose last cells lie past 2^32 -- flat
    offsets past 2^31 - 1 and 64-bit sort keys -- sampled at the last face, forward and backward."""
    from pytorch3d_b200 import _C
    F, R, C = 2 ** 20 + 1, 64, 1
    assert F * R * R * C > 2 ** 32 and _C.texture_atlas_key_bits(F, R)[1] == 8
    atlas = torch.zeros((F, R, R, C), dtype=torch.float32, device=DEV)
    atlas[-2:] = torch.rand(2, R, R, C, generator=torch.Generator().manual_seed(2)).to(DEV)
    K = 6
    p2f = torch.full((1, 1, 2, K), F - 1, dtype=torch.int64, device=DEV)
    p2f[0, 0, 1] = F - 2
    p2f[0, 0, 0, -1] = -1  # background: atlas[F-1, 0, 0] times 0
    g = torch.Generator().manual_seed(3)
    bary = torch.rand(1, 1, 2, K, 3, generator=g)
    bary[0, 0, 0, 0] = torch.tensor([0.999, 0.0, 0.001])  # cell (w_y, w_x) = (0, 63)
    bary[0, 0, 0, 1] = torch.tensor([0.0, 0.999, 0.001])  # (63, 0)
    bary = bary.to(DEV)
    got = _C.texture_atlas_forward(p2f, bary, atlas)
    # the chain on the last two faces, with the face indices shifted (background stays -1 and wraps to the last face)
    shifted = types.SimpleNamespace(pix_to_face=torch.where(p2f >= 0, p2f - (F - 2), p2f), bary_coords=bary)
    sub = atlas[-2:].clone().requires_grad_(True)
    want = chain_sample(shifted, sub)
    assert torch.equal(got, want) and float(got.abs().sum()) > 0
    grad_texels = torch.randn(1, 1, 2, K, C, generator=g).to(DEV)
    grad = _C.texture_atlas_backward(grad_texels, p2f, bary, atlas)
    (want * grad_texels).sum().backward()
    _close(grad[-2:], sub.grad, "grad of the last two faces")
    assert int(grad[:-2].count_nonzero()) == 0


def _atlas_pipeline(sample, H=48, W=80, R=4):
    """Rasterize a torus batch, sample a seeded per-face atlas with `sample`, shade with the fused Phong shading, blend
    with the fused softmax blend, take a loss; returns the image, the gradients of the vertices and the atlas, and the
    texels."""
    from pytorch3d_b200 import synthetic
    from pytorch3d_b200.blending import BlendParams, softmax_rgb_blend
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    from pytorch3d_b200.shading import phong_shading
    m = synthetic.torus_batch(2, 24, 24, seed=1, device=DEV)
    m.requires_grad_(True)
    verts = m.verts_packed()
    F = m.faces_packed().shape[0]
    atlas = torch.rand(F, R, R, 3, generator=torch.Generator().manual_seed(5)).to(DEV).requires_grad_(True)
    # no blur: every slot's barycentrics lie in its triangle, so every cell is in range for the chain
    p2f, zbuf, bary, dists = rasterize_meshes(m, (H, W), blur_radius=0.0, faces_per_pixel=4)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf, dists=dists)
    assert_cells_in_range(frags, atlas)
    texels = sample(frags, atlas)
    lights = types.SimpleNamespace(ambient_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   diffuse_color=torch.tensor([[0.6, 0.5, 0.4]], device=DEV),
                                   specular_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   location=torch.tensor([[0.5, 1.0, -1.0]], device=DEV))
    cameras = types.SimpleNamespace(get_camera_center=lambda: torch.zeros(1, 3, device=DEV))
    materials = types.SimpleNamespace(ambient_color=torch.ones(1, 3, device=DEV),
                                      diffuse_color=torch.ones(1, 3, device=DEV),
                                      specular_color=torch.ones(1, 3, device=DEV),
                                      shininess=torch.tensor([64.0], device=DEV))
    colors = phong_shading(m, frags, lights, cameras, materials, texels)
    img = softmax_rgb_blend(colors, frags, BlendParams(sigma=1e-4, gamma=1e-4))
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), verts.grad, atlas.grad, texels.detach()


@pytest.mark.gpu
def test_end_to_end_atlas_phong_softmax_matches_torch_chain(built_lib):
    got = _atlas_pipeline(fused_sample)
    want = _atlas_pipeline(chain_sample)
    assert torch.equal(got[3], want[3])  # the texels; shading and blending may round differently downstream
    _close(got[0], want[0], "image")
    for name, a, b in zip(("grad_verts", "grad_atlas"), got[1:3], want[1:3]):
        assert float(b.abs().max()) > 0, name
        _close(a, b, name)


@pytest.mark.gpu
def test_atlas_errors_and_workspace_on_the_device(built_lib):
    from pytorch3d_b200 import _C, _lib
    s = atlas_scene(2, 3, 4, 2, 4, 3, device=DEV)
    p2f, bary, atlas = s["pix_to_face"], s["bary"], torch.cat(s["atlases"])
    with pytest.raises(RuntimeError, match="atlas.*Float"):
        _C.texture_atlas_forward(p2f, bary, atlas.double())
    with pytest.raises(RuntimeError, match="Long"):
        _C.texture_atlas_forward(p2f.int(), bary, atlas)
    with pytest.raises(RuntimeError, match="atlas must be a CUDA tensor"):
        _C.texture_atlas_forward(p2f, bary, atlas.cpu())
    with pytest.raises(RuntimeError, match="grad_texels"):
        _C.texture_atlas_backward(s["grad_texels"][..., :2], p2f, bary, atlas)
    lib = _lib.load()
    S = 8 * 512 * 512 * 8
    narrow = lib.b200r_texture_atlas_workspace_bytes(8, 512, 512, 8, 559504, 4)
    wide = lib.b200r_texture_atlas_workspace_bytes(8, 512, 512, 8, 2 ** 28, 4)  # 64-bit keys
    assert narrow >= 16 * S and wide >= 24 * S  # two key buffers and two slot-index buffers, then the sort's storage
    assert lib.b200r_texture_atlas_workspace_bytes(0, 512, 512, 8, 10, 4) == 0
