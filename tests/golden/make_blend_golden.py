"""Writes tests/golden/reference_golden_blend*.npz: the outputs of the reference's own blending on the seeded scenes of
tests/test_blending.py, in the record format of make_reference_golden.py (tests/helpers.py: reference_record).

Parts (--parts, default both):
  cpu   reference_golden_blend.npz       the reference's C++ CPU sigmoid_alpha_blend op (forward, backward), and its
                                         softmax_rgb_blend / hard_rgb_blend run on the CPU from its own
                                         pytorch3d/renderer/blending.py (outputs and autograd gradients).  Needs the
                                         reference tree and oracle/_ref/ref_blend_cpu.so.
  cuda  reference_golden_blend_cuda.npz  the reference's CUDA sigmoid_alpha_blend kernels (forward, backward), built for
                                         sm_90a into oracle/_ref/ref_blend_cuda.so.  Needs a CUDA device.
Build the reference modules first: python oracle/build_ref_blend.py

    python tests/golden/make_blend_golden.py [--parts cpu,cuda] [OUT_DIR]
"""
import argparse
import importlib.util
import os
import sys
import types
from typing import Union

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from helpers import reference_record  # noqa: E402
from oracle import build_ref, build_ref_blend  # noqa: E402

EXACT_ROWS, SAMPLE_ROWS = 4, 1024


def put(store, case, arrays, lead, max_rows):
    for i, rec in enumerate(reference_record(arrays, lead, max_rows)):
        for field, v in rec.items():
            store["%s/%d/%s" % (case, i, field)] = v


def reference_blending_module():
    """The reference's pytorch3d/renderer/blending.py, imported with stand-ins for `pytorch3d._C` (only its sigmoid op
    uses it) and pytorch3d.common.datatypes."""
    path = os.path.join(build_ref.REF, "pytorch3d", "renderer", "blending.py")
    stubs = {n: types.ModuleType(n) for n in ("pytorch3d", "pytorch3d.common", "pytorch3d.common.datatypes")}
    stubs["pytorch3d"]._C = types.SimpleNamespace()
    stubs["pytorch3d.common.datatypes"].Device = Union[str, torch.device]
    saved = {n: sys.modules.get(n) for n in stubs}
    sys.modules.update(stubs)
    try:
        spec = importlib.util.spec_from_file_location("reference_blending", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    return mod


def cpu_part():
    import test_blending as tb
    ref = build_ref_blend.load(cuda=False)
    assert ref is not None, "build the reference first (oracle/build_ref_blend.py)"
    store = {}
    for args in tb.SIGMOID_CASES:
        dists, p2f, ga = tb.sigmoid_scene(*args)
        alphas = ref.sigmoid_alpha_blend(dists, p2f, args[4])
        grad = ref.sigmoid_alpha_blend_backward(ga, alphas, dists, p2f, args[4])
        put(store, tb.sigmoid_case(args) + "/cpu", [alphas, grad], 3, SAMPLE_ROWS)
    rb = reference_blending_module()
    for args in tb.SOFTMAX_CASES:
        colors, p2f, zbuf, dists, znear, zfar, grad = tb.softmax_scene(*args[:5], args[6])
        params = rb.BlendParams(sigma=args[4], gamma=args[5], background_color=(0.2, 0.4, 0.6))
        got = tb.softmax_with_grads(lambda c, p, z, d: rb.softmax_rgb_blend(c, tb.frags(p, z, d), params, znear, zfar),
                                    colors, p2f, zbuf, dists, grad)
        put(store, tb.softmax_case(args), got, 3, EXACT_ROWS)
    colors, p2f, zbuf, dists, grad = tb.reference_8x8_scene()
    params = rb.BlendParams(sigma=1e-3)
    got = tb.softmax_with_grads(lambda c, p, z, d: rb.softmax_rgb_blend(c, tb.frags(p, z, d), params), colors, p2f,
                                zbuf, dists, grad)
    put(store, "blend_softmax/reference_8x8", got, 3, EXACT_ROWS)
    colors, p2f, zbuf, dists, _, _, grad = tb.softmax_scene(2, 9, 13, 4, 1e-4, "scalar")
    c = colors.clone().requires_grad_(True)
    out = rb.hard_rgb_blend(c, tb.frags(p2f, zbuf, dists), rb.BlendParams(background_color=(0.2, 0.4, 0.6)))
    out.backward(grad)
    put(store, "blend_hard/2-9-13-4", [out.detach(), c.grad], 3, EXACT_ROWS)
    return store


def cuda_part():
    import test_blending as tb
    ref = build_ref_blend.load(cuda=True)
    assert ref is not None, "build the reference first (oracle/build_ref_blend.py)"
    assert torch.cuda.is_available(), "the reference's CUDA kernels need a CUDA device"
    dev = torch.device("cuda:0")
    store = {}
    for args in tb.SIGMOID_CASES + [tb.TORUS_SIGMOID]:
        if args[0] == "torus":
            p2f, _, _, dists = tb.torus_fragments(dev)
            ga = torch.randn(p2f.shape[:3], generator=torch.Generator().manual_seed(5)).to(dev)
            sigma = args[1]
        else:
            dists, p2f, ga = (t.to(dev) for t in tb.sigmoid_scene(*args))
            sigma = args[4]
        alphas = ref.sigmoid_alpha_blend(dists, p2f, sigma)
        grad = ref.sigmoid_alpha_blend_backward(ga, alphas, dists, p2f, sigma)
        put(store, tb.sigmoid_case(args) + "/cuda", [alphas, grad], 3, EXACT_ROWS)
    return store


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir", nargs="?", default=HERE)
    ap.add_argument("--parts", default="cpu,cuda", help="comma-separated subset of: cpu, cuda")
    a = ap.parse_args()
    torch.set_grad_enabled(True)
    for part in a.parts.split(","):
        store = {"cpu": cpu_part, "cuda": cuda_part}[part]()
        out = os.path.join(a.out_dir, "reference_golden_blend%s.npz" % ("_cuda" if part == "cuda" else ""))
        np.savez_compressed(out, **store)
        print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
        assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
