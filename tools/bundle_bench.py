"""Bundle adjustment of a posed image set: `bundle_adjust` (`ltr_bundle_adjust`) over the tracks of the tracks bench
scene with perturbed poses.

    python tools/bundle_bench.py [--images 64] [--neighbours 4] [--points 2000] [--lines 300] [--outliers 0.3]
                                 [--deg 0.3] [--shift 0.03] [--reps 10]

Data: the scene and pair ring of tools/tracks_bench.py (0.5 px of noise, --outliers of the observations moved 10 to
60 px, ground-truth matches); every image but image 0 has its pose perturbed by a rotation of --deg degrees and a
centre shift of --shift units (random directions), tracks at 8 px, image 0 fixed.  Device times are CUDA-event medians
of --reps calls after a warm-up, and the kernel time from ltr_profile_*.  Errors are medians over the images (rotation
in degrees, centre distance) and over the participating tracks (points; lines: the larger end-point distance to the
true segment's line), before and after.  The per-kernel times come from torch.profiler in a call of its own.  The
CPU comparison is one timed scipy.optimize.least_squares run (trf, finite-difference Jacobian with the problem's
sparsity) on the same residuals, parametrization and gauge from the same input, on the host.  Prints the GPU model
and power limit read in the same run, then one JSON line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
from scipy.optimize import least_squares
from scipy.sparse import coo_matrix
from scipy.spatial.transform import Rotation as Rot

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from linetr_b200 import _native as N, bundle as BA, synthetic as syn, tracks as TR   # noqa: E402
from triangulation_bench import gpu_info, ring_matches, time_cuda   # noqa: E402


def pose_errors(R, t, d):
    c = (np.einsum("nij,nij->n", R, d["R"]) - 1) / 2
    C, Cg = np.einsum("nji,nj->ni", R, -t), np.einsum("nji,nj->ni", d["R"], -d["t"])
    return float(np.median(np.degrees(np.arccos(np.clip(c, -1, 1)))[1:])), \
        float(np.median(np.linalg.norm(C - Cg, axis=1)[1:]))


def structure_errors(P, L, d, sel_p, sel_l, tracks):
    """Median point error and line error over the participating tracks (each track's truth: its first row's)."""
    n, m = len(d["points3d"]), len(d["segments3d"])
    op, ol = tracks.obs_p.cpu().numpy(), tracks.obs_l.cpu().numpy()
    top, tol = tracks.track_off_p.cpu().numpy(), tracks.track_off_l.cpu().numpy()
    tp = d["points3d"][op[top[:-1][:len(P)]] % n]
    ep = np.linalg.norm(P - tp, axis=1)[sel_p]
    S = d["segments3d"][ol[tol[:-1][:len(L)]] % m]
    u = S[:, 1] - S[:, 0]
    u = u / np.linalg.norm(u, axis=1, keepdims=True)
    el = []
    for e in range(2):
        w = L[:, e] - S[:, 0]
        el.append(np.linalg.norm(w - (w * u).sum(1, keepdims=True) * u, axis=1))
    return float(np.median(ep)), float(np.median(np.maximum(*el)[sel_l]))


def scipy_reference(d, R0, t0, tr, status_p, status_l, fixed=(0,)):
    """One timed scipy.optimize.least_squares run (trf, sparse Jacobian by finite differences) on the same residuals,
    camera parametrization and gauge, started from the same input.  Lines use the in-plane basis of their input
    direction (the model re-bases after every step).  -> (seconds, function evaluations, final cost)."""
    n = len(R0)
    get = lambda nm: tr[nm] if isinstance(tr, dict) else getattr(tr, nm).cpu().numpy()
    op, ol = np.asarray(tr["offsets_p"] if isinstance(tr, dict) else tr.offsets_p), \
        np.asarray(tr["offsets_l"] if isinstance(tr, dict) else tr.offsets_l)
    K = np.broadcast_to(d["K"], (n, 3, 3)) if np.ndim(d["K"]) == 2 else d["K"]
    C0 = np.einsum("nji,nj->ni", R0, -t0)
    rows = {}
    for kind, st, off in (("p", status_p, op), ("l", status_l, ol)):
        obs, toff, inl = get(f"obs_{kind}"), get(f"track_off_{kind}"), get(f"inlier_{kind}")
        tk, rr = [], []
        for j, k in enumerate(np.flatnonzero(st == BA.BA_IN)):
            o = obs[toff[k]:toff[k + 1]]
            o = o[inl[o] == 1]
            tk.append(np.full(len(o), j))
            rr.append(o)
        tk = np.concatenate(tk) if tk else np.zeros(0, np.int64)
        rr = np.concatenate(rr) if rr else np.zeros(0, np.int64)
        rows[kind] = (tk, rr, np.searchsorted(off, rr, side="right") - 1)
    part = np.zeros(n, bool)
    part[rows["p"][2]] = part[rows["l"][2]] = True
    free = [i for i in range(n) if i not in fixed and part[i]]
    col = np.full((n, 6), -1)
    nc = 0
    hold = BA._hold(R0, t0, list(fixed))
    for j, i in enumerate(free):
        for a in range(6):
            if not (len(fixed) == 1 and j == 0 and a == 3 + hold[i]):
                col[i, a] = nc
                nc += 1
    P0 = get("points3d")[:len(status_p)][status_p == BA.BA_IN]
    L0 = get("lines3d").reshape(-1, 6)[:len(status_l)][status_l == BA.BA_IN]
    dd = L0[:, 3:] - L0[:, :3]
    e = np.eye(3)[np.argmin(np.abs(dd), 1)]
    u1 = np.cross(dd, e)
    u1 /= np.linalg.norm(u1, axis=1, keepdims=True)
    u2 = np.cross(dd, u1)
    u2 /= np.linalg.norm(u2, axis=1, keepdims=True)
    kp = np.concatenate([k.reshape(-1, 2) for k in d["keypoints"]]).astype(np.float64)
    kl = np.concatenate([k.reshape(-1, 4) for k in d["klines"]]).astype(np.float64)
    tp, rp, ip = rows["p"]
    tl, rl, il = rows["l"]
    s = kl[rl]
    a, b, c = s[:, 1] - s[:, 3], s[:, 2] - s[:, 0], s[:, 0] * s[:, 3] - s[:, 2] * s[:, 1]
    nn = np.hypot(a, b)
    Kl = K[il]
    nv = np.stack([a / nn * Kl[:, 0, 0], b / nn * Kl[:, 1, 1], (a * Kl[:, 0, 2] + b * Kl[:, 1, 2] + c) / nn], 1)
    Kp, px = K[ip], kp[rp]
    npn = 3 * len(P0)

    def fun(x):
        dc = np.concatenate([x[:nc], [0.0]])[col]
        w = dc[:, :3]
        ww = (w * w).sum(1)[:, None, None]
        wx = np.zeros((n, 3, 3))
        wx[:, 0, 1], wx[:, 0, 2], wx[:, 1, 2] = -w[:, 2], w[:, 1], -w[:, 0]
        wx = wx - wx.transpose(0, 2, 1)
        Cay = ((1 - ww) * np.eye(3) + 2 * wx + 2 * w[:, :, None] * w[:, None, :]) / (1 + ww)
        R, C = Cay @ R0, C0 + dc[:, 3:]
        P = P0 + x[nc:nc + npn].reshape(-1, 3)
        q = x[nc + npn:].reshape(-1, 4)
        Xa = L0[:, :3] + u1 * q[:, :1] + u2 * q[:, 1:2]
        Xb = L0[:, 3:] + u1 * q[:, 2:3] + u2 * q[:, 3:4]
        Q = np.einsum("nij,nj->ni", R[ip], P[tp] - C[ip])
        out = [(Kp[:, 0, 0] * Q[:, 0] - (px[:, 0] - Kp[:, 0, 2]) * Q[:, 2]) / Q[:, 2],
               (Kp[:, 1, 1] * Q[:, 1] - (px[:, 1] - Kp[:, 1, 2]) * Q[:, 2]) / Q[:, 2]]
        for X in (Xa, Xb):
            Q = np.einsum("nij,nj->ni", R[il], X[tl] - C[il])
            out.append((nv * Q).sum(1) / Q[:, 2])
        return np.concatenate(out)

    npr, nlr = len(rp), len(rl)
    ri, ci = [], []
    for img, lm, width, base, r0 in ((ip, tp, 3, nc, 0), (ip, tp, 3, nc, npr), (il, tl, 4, nc + npn, 2 * npr),
                                     (il, tl, 4, nc + npn, 2 * npr + nlr)):
        r = r0 + np.arange(len(img))
        for a_ in range(6):
            cc = col[img, a_]
            ri.append(r[cc >= 0])
            ci.append(cc[cc >= 0])
        for k in range(width):
            ri.append(r)
            ci.append(base + width * lm + k)
    ri, ci = np.concatenate(ri), np.concatenate(ci)
    nx = nc + npn + 4 * len(L0)
    S = coo_matrix((np.ones(len(ri)), (ri, ci)), shape=(2 * npr + 2 * nlr, nx)).tocsr()
    t_0 = time.perf_counter()
    sol = least_squares(fun, np.zeros(nx), jac_sparsity=S, method="trf", x_scale="jac", ftol=1e-10)
    secs = time.perf_counter() - t_0
    return secs, int(sol.nfev), float((sol.fun ** 2).sum())


def kernel_breakdown(call):
    """Per-kernel device time (ms) of one call, from torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key.split("(")[0].split("::")[-1]
        if name.startswith("ba_"):
            dt = getattr(ev, "device_time_total", None)
            if dt is None:
                dt = ev.cuda_time_total
            out[name] = (round(dt / 1000.0, 3), int(ev.count))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--neighbours", type=int, default=4)
    ap.add_argument("--points", type=int, default=2000)
    ap.add_argument("--lines", type=int, default=300)
    ap.add_argument("--outliers", type=float, default=0.3)
    ap.add_argument("--deg", type=float, default=0.3)
    ap.add_argument("--shift", type=float, default=0.03)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bundle_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    V = args.images
    d = syn.make_line_map_set(0, V, args.points, args.lines, jitter_px=0.5, outlier_frac=args.outliers)
    pairs = np.array([(i, (i + k) % V) for i in range(V) for k in range(1, args.neighbours + 1)], dtype=np.int32)
    rng = np.random.default_rng(1)
    R, t = d["R"].copy(), d["t"].copy()
    for v in range(1, V):
        dR = Rot.from_rotvec(rng.normal(size=3) / np.sqrt(3) * np.deg2rad(args.deg)).as_matrix()
        C = -R[v].T @ t[v] + rng.normal(size=3) / np.sqrt(3) * args.shift
        R[v] = dR @ R[v]
        t[v] = -R[v] @ C
    res = ring_matches(d, pairs, dev)
    trk = TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], R, t, thresh=8, epi_thresh=8)
    call = lambda: BA.bundle_adjust(d["keypoints"], d["klines"], d["K"], R, t, trk)
    med, lo, hi = time_cuda(call, args.reps)
    N.profile_begin()
    out = call()
    kern = N.profile_end().get("bundle", (float("nan"), 0))
    per_kernel = kernel_breakdown(call)
    st = out.stats_dict()
    ntp, ntl = trk.n_tracks()
    sp, sl = out.status_p[:ntp].cpu().numpy(), out.status_l[:ntl].cpu().numpy()
    P0, L0 = trk.points3d[:ntp].cpu().numpy(), trk.lines3d[:ntl].cpu().numpy()
    P1, L1 = out.points3d[:ntp].cpu().numpy(), out.lines3d[:ntl].cpu().numpy()
    before = pose_errors(R, t, d) + structure_errors(P0, L0, d, sp == BA.BA_IN, sl == BA.BA_IN, trk)
    after = pose_errors(out.R.cpu().numpy(), out.t.cpu().numpy(), d) + \
        structure_errors(P1, L1, d, sp == BA.BA_IN, sl == BA.BA_IN, trk)
    sp_secs, sp_nfev, sp_cost = scipy_reference(d, R, t, trk, sp, sl)
    gpu = gpu_info()
    keys = ("rot_deg", "centre", "point", "line")
    print(f"{gpu}: {V} posed images, {len(pairs)} pairs, {args.points} keypoints and {args.lines} key lines per image, "
          f"{args.outliers:.0%} moved, poses perturbed {args.deg} deg / {args.shift}")
    print(f"  bundle_adjust call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}); kernels {kern[0]:.3f} ms in "
          f"{kern[1]} launches; "
          f"{st['iterations']} iterations, {st['accepted']} accepted, stop {st['stop_reason']}; cost "
          f"{st['initial_cost']:.1f} -> {st['final_cost']:.1f} over {st['n_obs']} rows of {st['n_tracks']} tracks")
    print("  kernels (ms, launches): " + ", ".join(f"{k} {v[0]:.3f} ({v[1]})" for k, v in per_kernel.items()))
    print(f"  scipy least_squares (trf, sparse Jacobian, host): {sp_secs:.2f} s, {sp_nfev} evaluations, cost "
          f"{sp_cost:.1f}")
    print("  median errors before -> after: " + ", ".join(f"{k} {b:.3e} -> {a:.3e}"
                                                          for k, b, a in zip(keys, before, after)))
    print(json.dumps({"gpu": gpu, "images": V, "pairs": len(pairs), "call_ms": med, "kernel_ms": kern[0],
                      "stats": st, "status_p": np.bincount(sp, minlength=4).tolist(),
                      "status_l": np.bincount(sl, minlength=4).tolist(),
                      "before": dict(zip(keys, before)), "after": dict(zip(keys, after)), "kernels_ms": per_kernel,
                      "scipy": {"seconds": sp_secs, "nfev": sp_nfev, "final_cost": sp_cost}}))


if __name__ == "__main__":
    main()
