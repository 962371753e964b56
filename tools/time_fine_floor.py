"""The fine pass of the north-star batch against its store floor (development aid).

    python tools/time_fine_floor.py [name ...]   # on a GPU; names: builds of tools/variant_time.py (default: the library)

The fine pass must write 28 B per slot of every pixel, -1 padding included, whatever the scene.  Translating the batch
off-screen empties every tile, so the same launch writes the same bytes and computes nothing: its time is the store floor
the kernel is judged against.  Each build is timed on both batches through the library's phase events, three times in
alternating order; the card's name and power limit are read in the same run.
"""
import ctypes
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch3d_b200 import _lib, synthetic  # noqa: E402

VARIANTS = os.path.join(ROOT, "tools", "_variants")
N, H, W, K = 8, 512, 512, 8
REPS, TIMED = 3, 30


def load(name):
    if name == "library":
        return _lib.load()
    lib = ctypes.CDLL(os.path.join(VARIANTS, "lib_%s.so" % name))
    for fn, (res, argt) in _lib.SIGNATURES.items():
        f = getattr(lib, fn)
        f.restype, f.argtypes = res, argt
    return lib


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "power limit unavailable (%s)" % e
    return "%s, %s" % (name, q)


def fine_ms(lib, fv, first, num):
    dev = fv.device
    F = fv.shape[0]
    p2f = torch.full((N, H, W, K), -1, dtype=torch.int64, device=dev)  # (a build may leave empty tiles unwritten)
    z, d = torch.empty((N, H, W, K), device=dev), torch.empty((N, H, W, K), device=dev)
    b = torch.empty((N, H, W, K, 3), device=dev)
    ws_bytes = lib.b200r_rasterize_meshes_workspace_bytes(F, N, H, W, 0)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def fwd():
        rc = lib.b200r_rasterize_meshes_forward(fv.data_ptr(), F, first.data_ptr(), num.data_ptr(), None, N, H, W, 0.0,
                                                K, 0, 0, 0, 0, 0, p2f.data_ptr(), z.data_ptr(), b.data_ptr(),
                                                d.data_ptr(), ws.data_ptr(), ws_bytes, 0, stream)
        assert rc == 0, lib.b200r_last_error()

    for _ in range(5):
        fwd()
    lib.b200r_set_profiling(1)
    buf = (ctypes.c_float * 3)()
    t = []
    for _ in range(TIMED):
        torch.cuda._sleep(400000)  # (the launch queue runs dry between samples: no overlap with the next call)
        fwd()
        lib.b200r_last_phase_ms(buf)
        t.append(buf[1])
    lib.b200r_set_profiling(0)
    t.sort()
    return t[len(t) // 2], int((p2f >= 0).sum())


def main():
    assert torch.cuda.is_available(), "tools/time_fine_floor.py times on a GPU"
    names = sys.argv[1:] or ["library"]
    dev = torch.device("cuda:0")
    print(card(), flush=True)
    m = synthetic.torus_batch(N, 187, 187, seed=0)
    fv = synthetic.face_verts_of(m).to(dev)
    off = fv.clone()
    off[..., 0] += 4.0  # every face right of the image: no tile is covered
    first, num = m.mesh_to_faces_packed_first_idx().to(dev), m.num_faces_per_mesh().to(dev)
    libs = {name: load(name) for name in names}
    res = {name: {"ns": [], "floor": []} for name in names}
    for rep in range(REPS):
        for name in (names if rep % 2 == 0 else names[::-1]):
            tf, hits = fine_ms(libs[name], fv, first, num)
            tz, zhits = fine_ms(libs[name], off, first, num)
            assert zhits == 0, "the off-screen batch still covers pixels"
            res[name]["ns"].append(tf)
            res[name]["floor"].append(tz)
            print("rep %d %-16s fine %.1f us  off-screen (store floor) %.1f us  ratio %.3f  hits %d" % (
                rep, name, tf * 1e3, tz * 1e3, tf / tz, hits), flush=True)
    alg = 28.0 * N * H * W * K
    for name in names:
        f, z = sorted(res[name]["ns"]), sorted(res[name]["floor"])
        print("%-16s fine %.1f us (%.1f-%.1f), floor %.1f us (%.1f-%.1f), fine / floor %.3f, floor writes %.2f TB/s" % (
            name, f[len(f) // 2] * 1e3, f[0] * 1e3, f[-1] * 1e3, z[len(z) // 2] * 1e3, z[0] * 1e3, z[-1] * 1e3,
            f[len(f) // 2] / z[len(z) // 2], alg / (z[len(z) // 2] * 1e-3) / 1e12), flush=True)


if __name__ == "__main__":
    main()
