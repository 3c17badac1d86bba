"""Phase clocks of the coupling-step kernel's final layer on one cfg-3 coupling (D = 784, H = 256, two residual blocks, 8 bins,
linear tails: 98 column tiles per 128-row tile).

Builds the library with NFK_STEP_CLOCKS (clock64 stamps in nfk_coupling_step_tc.cu, compiled out of the shipped library) into
its own output directory, loads it in place of nflows_b200/lib/libnfk_sm90.so, runs the coupling once to warm up and once
stamped, and prints one JSON line of medians in SM cycles together with the card's name and power limit.

    python scripts/step_phases.py [--rows N] [--out DIR | --lib LIB]

Stamps per column tile (by thread 0 of its warpgroup): t0 before the turn wait, t1 first slab landed, t2 last slab landed,
t3 MMAs retired, then per 64-row pass the sums staged (t4, t6) and the spline done (t5, t7)."""
import argparse
import ctypes
import glob
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "nflows_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-DNFK_STEP_CLOCKS"]


def build(out):
    """The instrumented library in `out` (objects and .so there; nothing under nflows_b200/ is written)."""
    os.makedirs(out, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    objs = [os.path.join(out, os.path.basename(s)[:-3] + ".o") for s in srcs]

    def compile_one(so):
        subprocess.run([NVCC] + FLAGS + ["-c", so[0], "-o", so[1]], check=True, cwd=CSRC)

    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(compile_one, zip(srcs, objs)))
    lib = os.path.join(out, "libnfk_sm90_clocks.so")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", lib] + objs, check=True)
    return lib


def power_limit_w(index=0):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def med(x):
    x = np.asarray(x, dtype=np.float64)
    return None if x.size == 0 else round(float(np.median(x)), 1)


def phases(buf, dims, nt, num_k):
    ctas, rounds, tiles, ns = dims
    rec = buf.reshape(ctas * rounds, 4 + tiles * ns)
    out = {k: [] for k in ("trunk", "turn_and_first_slab", "slab_wait_per_slab", "mma_per_tile", "mma_after_last_slab",
                           "staging", "spline_per_pass", "owner_period_per_tile", "final_layer_per_tile")}
    for r in rec:
        tr = r[:4].reshape(2, 2)
        if not np.all(tr > 0):
            continue
        out["trunk"] += list(tr[:, 1] - tr[:, 0])
        st = r[4:].reshape(tiles, ns)[:nt]
        if not np.all(st > 0):
            continue
        out["turn_and_first_slab"] += list(st[:, 1] - st[:, 0])
        out["slab_wait_per_slab"] += list((st[:, 2] - st[:, 1]) / max(num_k - 1, 1))
        out["mma_per_tile"] += list(st[:, 3] - st[:, 1])
        out["mma_after_last_slab"] += list(st[:, 3] - st[:, 2])
        out["staging"] += list(st[:, 4] - st[:, 3]) + list(st[:, 6] - st[:, 5])
        out["spline_per_pass"] += list(st[:, 5] - st[:, 4]) + list(st[:, 7] - st[:, 6])
        out["owner_period_per_tile"] += list(st[2:, 0] - st[:-2, 0])
        out["final_layer_per_tile"].append((st[:, 7].max() - tr[:, 1].min()) / nt)
    return {k: med(v) for k, v in out.items()}, len(out["final_layer_per_tile"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 19)
    ap.add_argument("--out", default=None, help="build directory of the instrumented library (default: a temporary one)")
    ap.add_argument("--lib", default=None, help="use this instrumented library (built before with --out) instead of building")
    args = ap.parse_args()
    lib_path = args.lib or build(args.out or tempfile.mkdtemp(prefix="nfk_step_clocks_"))

    from nflows_b200 import _native
    _native._LIB_PATH = lib_path              # before the first load
    import torch

    from nflows_b200 import config
    from nflows_b200 import kernels as K
    from nflows_b200.flows import recipes

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    flow = recipes.perturb_(recipes.rq_nsf(784)).eval()
    coupling = [m for m in flow.modules() if type(m).__name__ == "PiecewiseRationalQuadraticCouplingTransform"][0].to(dev)
    hidden = 256
    d_t = int(coupling.num_transform_features)
    x = torch.randn(args.rows, 784, device=dev)
    with torch.no_grad():
        coupling(x)
        torch.cuda.synchronize()
        K.TIMELINE = []
        coupling(x)
        torch.cuda.synchronize()
        tags = sorted({t[0] for t in K.TIMELINE})
        step_ms = sum(t[2].elapsed_time(t[3]) for t in K.TIMELINE if t[0] == "rq_coupling_step")
        K.TIMELINE = None
    assert "rq_coupling_step" in tags, tags
    lib = ctypes.CDLL(lib_path)
    dims = (ctypes.c_int32 * 4)()
    assert lib.nfk_step_clocks(None, dims) == 0
    dims = tuple(dims)
    buf = np.zeros(dims[0] * dims[1] * (4 + dims[2] * dims[3]), dtype=np.int64)
    assert lib.nfk_step_clocks(buf.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)), (ctypes.c_int32 * 4)()) == 0
    nt = (d_t + 3) // 4
    med_cycles, records = phases(buf, dims, nt, hidden // 32)
    print(json.dumps({"workload": "cfg-3 RQ coupling D=784 H=256 K=8 linear tails, coupling-step kernel",
                      "rows": args.rows, "column_tiles": nt, "stamped_row_tiles": records, "cycles_median": med_cycles,
                      "rq_coupling_step_ms": round(step_ms, 3), "block_rows": config.coupling_block_rows,
                      "gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}))


if __name__ == "__main__":
    main()
