#!/usr/bin/env python
"""Count the work of the backward render at the bench workload, on the CPU: work items, walked 32-record chunks and the
(record, sub-tile) pairs whose ten moments go to L2 (step 2 of render_bwd_body, one flush slot each).

The CPU oracle (oracle/c_oracle.py) runs the forward of bench.build_scene's cloud for each view; its per-tile lists (the
reference's 3-sigma tile rectangles, (depth, index) order) are then replayed with the reference's compositing rules on every
8x4 sub-tile, the work item of the default backward (PPL 1).  An item walks the records before the largest n_contrib of its
pixels; a record of that walk is a pair when at least one of the item's pixels composites it (power <= 0, alpha >= 1/255,
position before the pixel's n_contrib).  The product bins by tighter opacity-aware boxes: its tile lists and walked chunks
differ a little, its pairs do not.

    python tools/bwd_reduction_count.py [--workload cfg2] [--views 0,1,...]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import c_oracle  # noqa: E402

TILE, SUB_W, SUB_H, CHUNK = 16, 8, 4, 32
ALPHA_MIN, ALPHA_MAX, T_STOP = 1.0 / 255.0, 0.99, 1e-4


def count_view(a, cloud, cam):
    bg = np.ones(3, np.float32)
    r = c_oracle.forward(**bench.cam_settings(cam, a, bg), means3D=cloud["means3D"], opacities=cloud["opacities"],
                         shs=cloud["shs"], scales=cloud["scales"], rotations=cloud["rotations"], dtype=np.float32)
    st = r.state()
    r.close()
    H = W = a.res
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    px, py = st["px"].astype(np.float64), st["py"].astype(np.float64)
    conic = st["conic"].astype(np.float64)
    opac = np.asarray(cloud["opacities"], np.float64).reshape(-1)
    depth = st["depth"]
    rect = st["rect"]
    nx, ny = np.maximum(rect[:, 2] - rect[:, 0], 0), np.maximum(rect[:, 3] - rect[:, 1], 0)
    cnt = nx * ny
    g_of = np.repeat(np.arange(len(cnt)), cnt)
    k = np.arange(len(g_of)) - np.repeat(np.cumsum(cnt) - cnt, cnt)          # instance number within its Gaussian
    tile = (rect[g_of, 1] + k // np.maximum(nx[g_of], 1)) * gx + rect[g_of, 0] + k % np.maximum(nx[g_of], 1)
    order = np.lexsort((g_of, depth[g_of], tile))
    tile, g_of = tile[order], g_of[order]
    starts = np.searchsorted(tile, np.arange(gx * gy))
    ends = np.searchsorted(tile, np.arange(gx * gy), side="right")

    # pixel offsets of a tile, sub-tile major: sub s = (sub row) * 2 + (sub column), 32 pixels each
    ox = np.array([(s & 1) * SUB_W + (i & 7) for s in range(8) for i in range(32)], np.float64)
    oy = np.array([(s >> 1) * SUB_H + (i >> 3) for s in range(8) for i in range(32)], np.float64)
    walks, pairs, chunks, empty_chunks, pops = [], 0, 0, 0, []
    for t in range(gx * gy):
        s, e = starts[t], ends[t]
        if s == e:
            continue
        gs = g_of[s:e]
        pops.append(e - s)
        X = (t % gx) * TILE + ox
        Y = (t // gx) * TILE + oy
        inside = (X < W) & (Y < H)
        dx = px[gs, None] - X[None, :]
        dy = py[gs, None] - Y[None, :]
        power = -0.5 * (conic[gs, 0, None] * dx * dx + conic[gs, 2, None] * dy * dy) - conic[gs, 1, None] * dx * dy
        alpha = np.minimum(ALPHA_MAX, opac[gs, None] * np.exp(np.minimum(power, 0.0)))
        valid = (power <= 0) & (alpha >= ALPHA_MIN) & inside[None, :]
        Tafter = np.cumprod(np.where(valid, 1.0 - alpha, 1.0), axis=0)
        comp = valid & (Tafter >= T_STOP)                       # composited: before the pixel's early termination
        idx = np.arange(e - s)[:, None] + 1
        last = np.max(np.where(comp, idx, 0), axis=0)           # n_contrib of every pixel
        for sub in range(8):
            cols = slice(32 * sub, 32 * sub + 32)
            n = int(last[cols].max())
            walks.append(n)
            if n == 0:
                continue
            hit = comp[:n, cols].any(axis=1)
            pairs += int(hit.sum())
            nc = (n + CHUNK - 1) // CHUNK
            chunks += nc
            empty_chunks += nc - int(np.count_nonzero(np.add.reduceat(hit, np.arange(0, n, CHUNK))))
    walks = np.array(walks)
    walked = walks[walks > 0]
    return dict(nonempty_tiles=len(pops), items=len(walks), items_walked=int(len(walked)), chunks_walked=chunks,
                chunks_without_pair=empty_chunks, pairs=pairs, scalar_reductions=10 * pairs,
                walk_mean=float(walked.mean()) if len(walked) else 0.0,
                walk_p99=float(np.percentile(walked, 99)) if len(walked) else 0.0,
                median_tile_records=float(np.median(pops)) if pops else 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--views", default="0", help="comma-separated camera numbers of the bench's view set, or 'all'")
    ap.add_argument("--opacity", default="trained", choices=["trained", "init"])
    args = ap.parse_args()
    w = bench.WORKLOADS[args.workload]
    a = argparse.Namespace(sh_degree=3, opacity=args.opacity, seed=0, workload=args.workload,
                           **{k: w[k] for k in ("points", "res", "views_per_gpu", "views")})
    cloud, cams, _ = bench.build_scene(a)
    views = range(len(cams)) if args.views == "all" else [int(v) for v in args.views.split(",")]
    c_oracle.set_threads(bench.host_threads())
    print("%s: %s" % (args.workload, bench.workload_name(a)))
    for v in views:
        c = count_view(a, cloud, cams[v])
        print("view %d: " % v + ", ".join("%s %s" % (k, ("%.1f" % x) if isinstance(x, float) else x) for k, x in c.items()), flush=True)


if __name__ == "__main__":
    main()
