"""Host-side count of the work the tensor-core tile kernels do on the bench workload (cfg2: B=16, 256x256, k=5, C=256),
with and without skipping the MMA tiles of inactive 16-pixel group rows.

    python tools/tile_work.py [--flow smooth|iid|both] [--seed N] [--B 16] [--H 256] [--W 256] [--k 5] [--C 256] [--cn 128]

Flows come from bench.py's two families (smooth = x16 bilinear up-sampling of U(-8,8), iid = U(-8,8)) drawn with their
own seed, so these are statistics of the family, not of the bench's exact tensors.  The tap arithmetic is the kernels'
(axis_tap in fp32, clamped windows), the footprint is group_bbox's and the steps are the kernels' row-major walk over the
footprint.  A pixel is active in a K-step (16 positions) when window_meets_step holds (tile_window.cuh); irregular
pixels never are.  Warps of 32 pixels, mma.sync m16n8k16, ldmatrix .x4 = 512 B.

Channels-last forward (k_local_attn_fwd_tc_cl), counted per CTA over C / CN passes of CN channels and 32-position steps
(two K-steps each):
  MMAs      CN / 8 per m-tile (16 pixels) active in a K-step
  ldmatrix  per K-step, 1 A per active m-tile, CN / 16 B per MMA warp with an active m-tile
  slab      bytes stored into the weight slabs: the pixel warps' window entries (2 B each, scattered), the MMA warps'
            zero fill (64 B per slab row of an m-tile active in either K-step of the step)
  barriers  per step FULL and FREE (256 threads each)
Backward, per CTA-step (16-position steps, one pass of 256 channels): P GEMM per warp: 16 k-steps x (2 A + 1 B)
ldmatrix, 4 MMAs; GS GEMM per group row: 4 warps x (1 + 4) ldmatrix, 4 x 8 MMAs; skip: inactive m-tiles / group rows
drop theirs, a step without any drops all.

grad_source reductions of the backward, per CTA-step.  A position of the step receives a partial sum when some active
pixel's clamped window covers it (every window entry is taken as nonzero).  Each warp adds its 64 channels of the
16 positions, 8 positions (one half of the segment) per warp instruction:
  bf16x2     (before) 8 instructions per warp and half with a covered position; each lane adds 4 B, so a position costs
             one half-used 32-B sector per instruction: 32 sector operations per covered position
  bf16x8     (now) the quad regroups its fragments so a lane holds 8 consecutive channels: 2 instructions per warp and
             half, 64 contiguous bytes per position each, so 16 full-sector operations per covered position
  fp32 pairs positions on the image border go to the fp32 scratch as before: 8 instructions per warp and half, one full
             sector per position each
"""
import argparse

import numpy as np

SEG, GW, GH = 16, 16, 8
LDSM = 512


def make_flow(kind, B, H, W, seed):
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    if kind == "smooth":
        coarse = torch.rand(B, 2, H // 16, W // 16, generator=g) * 16 - 8
        flow = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=True)
    else:
        flow = torch.rand(B, 2, H, W, generator=g) * 16 - 8
    return flow.float().numpy()


def taps(flow, coord, k, dim):
    """fl[j] = floor((flow + (j - k//2)) + coord) in fp32 (axis_tap), for j = 0..k-1"""
    fl = [np.floor((flow + np.float32(j - k // 2)) + coord.astype(np.float32)).astype(np.int64) for j in range(k)]
    regular = np.all([fl[j] == fl[0] + j for j in range(k)], axis=0)
    lo = np.clip(fl[0], 0, dim - 1)
    hi = np.clip(fl[k - 1] + 1, 0, dim - 1)
    return fl[0], regular, lo, hi


def count(flow, k, C, CN):
    B, _, H, W = flow.shape
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    X0, rx, bxlo, bxhi = taps(flow[:, 0], xs[None], k, W)
    Y0, ry, bylo, byhi = taps(flow[:, 1], ys[None], k, H)
    regular = rx & ry
    cx0, cx1 = np.clip(X0, 0, W - 1), np.clip(X0 + k, 0, W - 1)
    cy0, cy1 = np.clip(Y0, 0, H - 1), np.clip(Y0 + k, 0, H - 1)
    inimg = np.ones((B, H, W), bool)
    st = dict(groups=0, steps=[], entries=0, rows_on=0, warps_on=0, empty=0,
              f_steps=0, f_mma=0, f_ldsm=0, f_scatter=0, f_zero=0, f_bar=0, b_mma=[0, 0], b_ldsm=[0, 0], red_ins=[0, 0], red_sec=[0, 0], f32_ins=0, f32_sec=0)
    for b in range(B):
        for gy in range(0, H, GH):
            for gx in range(0, W, GW):
                sl = (b, slice(gy, gy + GH), slice(gx, gx + GW))
                pad = lambda a, v: np.pad(a[sl], ((0, GH - a[sl].shape[0]), (0, GW - a[sl].shape[1])), constant_values=v).reshape(-1)
                valid = pad(inimg, False)
                bx0, bx1 = bxlo[sl].min(), bxhi[sl].max()
                by0, by1 = bylo[sl].min(), byhi[sl].max()
                sx = np.arange(bx0, bx1 + 1, SEG)
                sy = np.arange(by0, by1 + 1)
                y = np.repeat(sy, len(sx))[:, None]
                x = np.tile(sx, len(sy))[:, None]
                reg = pad(regular, False) & valid
                a_x0, a_x1, a_y0, a_y1 = (pad(a, 0)[None] for a in (cx0, cx1, cy0, cy1))
                act = reg[None] & (a_y0 <= y) & (y <= a_y1) & (a_x0 < x + SEG) & (a_x1 >= x)     # [steps, 128]
                ent = np.clip(np.minimum(a_x1, x + SEG - 1) - np.maximum(a_x0, x) + 1, 0, None) * act
                rows = act.reshape(len(y), 8, 16).any(axis=2)                                     # [steps, group rows]
                n, nr = len(y), rows.sum(axis=1)
                st["groups"] += 1
                st["steps"].append(n)
                st["entries"] += ent.sum()
                st["rows_on"] += nr.sum()
                st["warps_on"] += rows.reshape(n, 4, 2).any(axis=2).sum()
                st["empty"] += (nr == 0).sum()
                wtiles = rows.reshape(n, 4, 2)
                # forward: 32-position steps, K-steps x and x + 16, C / CN passes that repeat the same walk
                passes = C // CN
                hx = np.arange(bx0, bx1 + 1, 2 * SEG)
                n2 = len(sy) * len(hx)
                y2 = np.repeat(sy, len(hx))[:, None, None]
                x2 = np.tile(hx, len(sy))[:, None, None] + np.array([0, SEG])[None, :, None]       # [steps, 2, 1]
                act2 = reg[None, None] & (a_y0[None] <= y2) & (y2 <= a_y1[None]) & (a_x0[None] < x2 + SEG) & (a_x1[None] >= x2)
                ent2 = (np.clip(np.minimum(a_x1[None], x2 + SEG - 1) - np.maximum(a_x0[None], x2) + 1, 0, None) * act2).sum()
                tiles2 = act2.reshape(n2, 2, 8, 16).any(axis=3)                                 # [steps, K-steps, m-tiles]
                st["f_steps"] += passes * n2
                st["f_mma"] += passes * (CN // 8) * tiles2.sum()
                st["f_ldsm"] += passes * (tiles2.sum() + (CN // 16) * tiles2.reshape(n2, 2, 4, 2).any(axis=3).sum()) * LDSM
                st["f_scatter"] += passes * 2 * ent2
                st["f_zero"] += passes * 16 * 2 * (2 * SEG) * tiles2.any(axis=1).sum()
                st["f_bar"] += passes * 2 * n2
                # backward, one pass of 256 channels
                st["b_mma"][0] += n * (4 * 16 * 4 + 8 * 32)
                st["b_ldsm"][0] += n * (4 * 16 * 3 + 8 * 20) * LDSM
                st["b_mma"][1] += 16 * 2 * nr.sum() + 32 * nr.sum()
                st["b_ldsm"][1] += (16 * (nr.sum() + wtiles.any(axis=2).sum()) + 20 * nr.sum()) * LDSM
                # grad_source reductions: positions x + e of the step that an active pixel's window covers
                pos = x + np.arange(SEG)[None]                                                    # [steps, 16]
                cov = (act[:, None, :] & (a_x0[:, None, :] <= pos[:, :, None])
                       & (pos[:, :, None] <= a_x1[:, None, :])).any(axis=2)
                border = (y == 0) | (y == H - 1) | (pos == 0) | (pos == W - 1)
                inner, edge = cov & ~border, cov & border
                halves, ehalves = inner.reshape(n, 2, 8).any(axis=2).sum(), edge.reshape(n, 2, 8).any(axis=2).sum()
                st["red_ins"][0] += 4 * 8 * halves
                st["red_ins"][1] += 4 * 2 * halves
                st["red_sec"][0] += 32 * inner.sum()
                st["red_sec"][1] += 16 * inner.sum()
                st["f32_ins"] += 4 * 8 * ehalves
                st["f32_sec"] += 32 * edge.sum()
    return st


def report(kind, st):
    steps = np.array(st["steps"])
    n = steps.sum()
    print(f"== {kind} flow: {st['groups']} groups of 16x8 pixels")
    print(f"steps per group (one pass)          mean {steps.mean():.1f}  p90 {np.percentile(steps, 90):.0f}  max {steps.max()}")
    print(f"window entries in the dense slab    {100 * st['entries'] / (n * 128 * SEG):.1f} %")
    print(f"active 16-pixel group rows          {100 * st['rows_on'] / (n * 8):.1f} %")
    print(f"active warps (32 pixels)            {100 * st['warps_on'] / (n * 4):.1f} %")
    print(f"steps without any active pixel      {100 * st['empty'] / n:.1f} %")
    g = st["groups"]
    print(f"forward per CTA ({st['C']} channels in passes of {st['CN']}): {st['f_steps'] / g:.1f} steps, {st['f_mma'] / g:.0f} MMAs, "
          f"ldmatrix {st['f_ldsm'] / g / 1024:.1f} KB, slab stores {st['f_scatter'] / g / 1024:.1f} KB scattered + "
          f"{st['f_zero'] / g / 1024:.1f} KB zero fill, {st['f_bar'] / g:.0f} barriers")
    print(f"forward per CTA-step: {st['f_mma'] / st['f_steps']:.1f} MMAs, ldmatrix {st['f_ldsm'] / st['f_steps'] / 1024:.1f} KB")
    for name, m, l in (("backward", st["b_mma"], st["b_ldsm"]),):
        print(f"{name:9s} per CTA-step   MMAs {m[0] / n:7.1f} -> {m[1] / n:7.1f}   ldmatrix {l[0] / n / 1024:6.1f} KB -> {l[1] / n / 1024:6.1f} KB"
              f"   ({100 * (1 - m[1] / m[0]):.0f} % / {100 * (1 - l[1] / l[0]):.0f} % skipped)")
    ri, rs = st["red_ins"], st["red_sec"]
    print(f"grad_source per CTA-step  bf16 reductions {ri[0] / n:5.1f} -> {ri[1] / n:5.1f} warp instructions, "
          f"{rs[0] / n:6.1f} -> {rs[1] / n:6.1f} sector operations (bf16x2 -> bf16x8)")
    print(f"                          border fp32 pairs {st['f32_ins'] / n:5.1f} warp instructions, {st['f32_sec'] / n:6.1f} sector operations")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--flow", default="both", choices=["smooth", "iid", "both"])
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--W", type=int, default=256)
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--C", type=int, default=256)
    ap.add_argument("--cn", type=int, default=128, choices=[64, 128], help="channels per forward pass")
    a = ap.parse_args()
    for kind in (["smooth", "iid"] if a.flow == "both" else [a.flow]):
        st = count(make_flow(kind, a.B, a.H, a.W, a.seed), a.k, a.C, a.cn)
        st.update(C=a.C, CN=a.cn)
        report(kind, st)


if __name__ == "__main__":
    main()
