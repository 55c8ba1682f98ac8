#!/usr/bin/env python
"""Time Pangu's block GEMMs one launch at a time, on both epilogue paths of the wgmma GEMM (gemm2.cuh).

    python tools/time_pangu_gemms.py [--members 1 4] [--iters 50] [--paths staged fragment] [--kscan] [--out result.json]

Each GEMM runs through libskyrim_b200_probe.so (oracle/gemm_probe.py) at the full 721 x 1440 token grids (C = 192 with
M = 521,280 tokens per member, C = 384 with M = 131,040), on random fp16 operand images made on the device:
  qkv    N = 3C, K = C,  window-image scatter (fragment path only: it has no staged form)
  proj   N = C,  K = C,  LayerNorm + residual into the fp16 token image (CTA pairs at C = 384)
  fc1    N = 4C, K = C,  GELU into the fp16 hidden image
  fc2    N = C,  K = 4C, LayerNorm + residual into the fp16 token image (CTA pairs at C = 384)
CUDA events around --iters back-to-back launches after five warm-up launches.  The two paths of a GEMM are timed in
turn, --rounds times (a power-limited card's clocks drift over a run), and the median counts.  Per GEMM and path it
prints us per launch, TFLOP/s (2 M N K over the time), the tile count and us per tile per SM (time x SMs / tiles).

It also times Pangu's fused MLP (mlp_fused.cuh: fc1, GELU and fc2 per row tile, the hidden activation in shared memory; CTA
pairs at C = 384) against fc1 + fc2 of the fragment path launched back to back on the same operands, alternated --rounds
times:
  mlp    fused against fc1_fc2, us per launch (pair) and TFLOP/s of the 4 M C^2 x 2 FLOPs of both GEMMs.

--kscan times fc1's tile grid (N = 4C) at K = C, 2C and 4C on the staged path: the same tiles with more k-blocks.  The
least-squares line through (k-blocks per tile, us per tile) splits a tile's time into the main loop's cost per k-block
(slope) and a fixed cost per tile (intercept).

The card's name, power limit and maximum SM clock are printed with the numbers (the times depend on them).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE = 16384
BN = 192
# sky_probe_gemm epilogue ids of the fragment path (gemm_probe.cu): EPI_F16_GELU_IMG / EPI_LN_IMG wrapped in FragEpi
EPI_F16_GELU_IMG_FRAG, EPI_LN_IMG_FRAG = 18, 19
MLP = 4   # sky_probe_gemm kernel id of the fused MLP (gemm_probe.cu SKY_PROBE_MLP)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--paths", nargs="+", default=["staged", "fragment"], choices=["staged", "fragment"])
    ap.add_argument("--kscan", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_pangu_gemms.py measures on the GPU and found none")
    from bench import gpu_identity
    from oracle import gemm_probe as gp
    from oracle import pangu_kernels_ref as pk
    from skyrim_b200.config import pangu_full

    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    epi_ids = {"staged": {"fc1": gp.EPI_F16_GELU_IMG, "ln": gp.EPI_LN_IMG}}
    if "fragment" in args.paths:
        epi_ids["fragment"] = {"fc1": EPI_F16_GELU_IMG_FRAG, "ln": EPI_LN_IMG_FRAG}
    res = {"gpu": gpu_identity(0), "sms": sms, "iters": args.iters, "gemms": [], "kscan": []}
    print(json.dumps(res["gpu"]), flush=True)

    def image(rows, nkb):
        """random fp16 tile image of `rows` rows and nkb k-blocks (values in [-1, 1))"""
        return torch.empty(-(-rows // 128) * nkb * TILE // 2, dtype=torch.float16, device=dev).uniform_(-1.0, 1.0)

    def weights(n, k):
        return torch.empty(n * k, dtype=torch.float16, device=dev).uniform_(-1.0, 1.0).mul_(float(1.0 / np.sqrt(k)))

    def vec(n, lo, hi):
        return torch.empty(n, dtype=torch.float32, device=dev).uniform_(lo, hi)

    def nbytes(t):
        return t.numel() * t.element_size()

    def time_case(*cases):
        """us per launch of `cases` one after the other"""
        for _ in range(5):
            for case in cases:
                rc, msg = gp.launch(case)
                assert rc == 0, msg
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            for case in cases:
                gp.launch(case)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.iters

    def report(name, path, C, B, M, N, K, us, tiles):
        rec = {"gemm": name, "path": path, "C": C, "members": B, "M": M, "N": N, "K": K, "us": round(us, 1),
               "tflops": round(2.0 * M * N * K / us * 1e-6, 1), "tiles": tiles, "k_blocks": K // 64,
               "us_per_tile": round(us * sms / tiles, 3)}
        print(json.dumps(rec), flush=True)
        return rec

    def gemm_case(kernel, epi, N, M, a, a_nkb, w, **kw):
        return gp.make_case(kernel=kernel, epi=epi, block_n=BN, n=N, n_valid=N, batches=1, grid_sms=0, nseg=1, m=M,
                            a=[a.data_ptr()], a_bytes=[nbytes(a)], a_batch_stride=[0], a_nkb=[a_nkb], w=w.data_ptr(),
                            w_bytes=nbytes(w), w_batch_stride=0, num_kb=a_nkb, w_rep=0, **kw)

    for g in pk.grids(pangu_full()):
        C, nkb = g.C, g.C // 64
        ln_kernel = gp.W if C == BN else gp.PAIR
        for B in args.members:
            M = B * g.T
            mt = -(-M // 128)
            x, hid = image(M, nkb), image(M, 4 * nkb)
            att = image(M, nkb)
            w_qkv, w_proj, w_fc1, w_fc2 = weights(3 * C, C), weights(C, C), weights(4 * C, C), weights(C, 4 * C)
            b3, bias, b4 = vec(3 * C, -0.1, 0.1), vec(C, -0.1, 0.1), vec(4 * C, -0.1, 0.1)
            gamma, beta = vec(C, 0.9, 1.1), vec(C, -0.1, 0.1)
            ln = dict(hi=x.data_ptr(), img_bytes=nbytes(x), img_nkb=nkb, bias=bias.data_ptr(), gamma=gamma.data_ptr(),
                      beta=beta.data_ptr(), vec_floats=C, eps=1e-5)
            # qkv: the window image (three parts, one 144-row tile per window and head pair each)
            wt = B * g.nWin * g.pairs
            qkv = torch.empty(3 * wt * pk.TILE_B // 2, dtype=torch.float16, device=dev)
            case = gemm_case(gp.W, gp.EPI_QKV_WIN, 3 * C, M, x, nkb, w_qkv, hi=qkv.data_ptr(), img_bytes=nbytes(qkv),
                             bias=b3.data_ptr(), vec_floats=3 * C, geo=g.probe_geo(), roll=1, pairs=g.pairs,
                             part_stride=wt * pk.TILE_B)
            res["gemms"].append(report("qkv", "fragment", C, B, M, 3 * C, C, time_case(case), mt * 3 * C // BN))
            del qkv
            for name, N, K in (("proj", C, C), ("fc1", 4 * C, C), ("fc2", C, 4 * C)):
                cases = {}
                for path in args.paths:
                    ids = epi_ids[path]
                    if name == "proj":
                        cases[path] = gemm_case(ln_kernel, ids["ln"], C, M, att, nkb, w_proj, **ln)
                    elif name == "fc1":
                        cases[path] = gemm_case(gp.W, ids["fc1"], N, M, x, nkb, w_fc1, hi=hid.data_ptr(), img_bytes=nbytes(hid),
                                                img_nkb=4 * nkb, bias=b4.data_ptr(), vec_floats=N)
                    else:
                        cases[path] = gemm_case(ln_kernel, ids["ln"], C, M, hid, 4 * nkb, w_fc2, **ln)
                times = {path: [] for path in args.paths}
                for _ in range(args.rounds):
                    for path in args.paths:
                        times[path].append(time_case(cases[path]))
                for path in args.paths:
                    res["gemms"].append(report(name, path, C, B, M, N, K, float(np.median(times[path])), mt * N // BN))
            # the fused MLP against fc1 + fc2 on the fragment path: W1 packed at BLOCK_N 64 for the fused kernel (the
            # weights are random, so a different packing of the same values is not needed for the timing)
            fc1 = gemm_case(gp.W, EPI_F16_GELU_IMG_FRAG, 4 * C, M, x, nkb, w_fc1, hi=hid.data_ptr(), img_bytes=nbytes(hid),
                            img_nkb=4 * nkb, bias=b4.data_ptr(), vec_floats=4 * C)
            fc2 = gemm_case(ln_kernel, EPI_LN_IMG_FRAG, C, M, hid, 4 * nkb, w_fc2, **ln)
            fused = gp.make_case(kernel=MLP, block_n=BN, n=C, n_valid=C, batches=1, grid_sms=0, m=M, w=w_fc1.data_ptr(),
                                 w_bytes=nbytes(w_fc1), b_hi=w_fc2.data_ptr(), b_bytes=nbytes(w_fc2), add=b4.data_ptr(),
                                 add_bytes=nbytes(b4), **ln)
            times = {"fc1_fc2": [], "fused": []}
            for _ in range(args.rounds):
                times["fc1_fc2"].append(time_case(fc1, fc2))
                times["fused"].append(time_case(fused))
            for path, t in times.items():
                rec = report("mlp", path, C, B, M, 4 * C, 2 * C, float(np.median(t)), mt)
                rec["share_of_989_tflops"] = round(rec["tflops"] / 989.0, 3)
                res["gemms"].append(rec)
            del x, hid, att
            torch.cuda.empty_cache()
        if args.kscan:
            M = g.T
            mt = -(-M // 128)
            hid = image(M, 4 * nkb)
            b4 = vec(4 * C, -0.1, 0.1)
            pts = []
            for mult in (1, 2, 4):
                K = mult * C
                a, w = image(M, K // 64), weights(4 * C, K)
                case = gemm_case(gp.W, gp.EPI_F16_GELU_IMG, 4 * C, M, a, K // 64, w, hi=hid.data_ptr(), img_bytes=nbytes(hid),
                                 img_nkb=4 * nkb, bias=b4.data_ptr(), vec_floats=4 * C)
                r = report("fc1_kscan", "staged", C, 1, M, 4 * C, K, time_case(case), mt * 4 * C // BN)
                pts.append((K // 64, r["us_per_tile"]))
                del a, w
            kb, ut = np.array(pts, float).T
            slope, icept = np.polyfit(kb, ut, 1)
            fit = {"C": C, "points": pts, "us_per_k_block": round(float(slope), 3), "us_fixed_per_tile": round(float(icept), 3),
                   "fixed_share_at_K=C": round(float(icept / ut[0]), 3)}
            print(json.dumps({"kscan_fit": fit}), flush=True)
            res["kscan"].append(fit)
            del hid
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
