"""Editing directions read from the UNet bottleneck h without training (`--h_directions`).

h-space is close to linear and homogeneous across images, so a direction for an attribute can be taken from the
statistics of h over many samples, one set per timestep of the generative grid:

  pca        the top K principal components of h.  The centred sample Gram G = X_c X_c^T (ops.h_gram, n x n, where
             the d x d covariance of d = C h w features is out of reach) is decomposed on the host in fp64
             (numpy.linalg.eigh); component k is v_k = X_c^T u_k / sqrt(λ_k) (ops.h_combine), a unit vector, stored
             as d_k = v_k sqrt(λ_k / (n - 1)): α = 1 moves h one standard deviation along it.
  mean_diff  d = μ₊ - μ₋, the mean h of images with the attribute minus that of images without it, unscaled: α = 1
             moves the negative set's mean onto the positive one.

Signs are fixed deterministically: at the first step (the largest t) each component's largest-|value| entry is made
positive, at every later step its dot product with the same component at the previous step is made >= 0.

An edit applies h2 = c0 h + α d_t at every edit step (UNetEngine.sample(h_direction=...)).  The file is one
torch.save dict per direction (pc<k>.pth, mean_diff.pth) holding d_t for every t of the grid; h_directions.tsv sums up
the run.
"""
import math
import os

import numpy as np
import torch

FORMAT = "asyrp_h_direction"


def _kernels(gram, combine):
    if gram is None or combine is None:
        from . import ops
        return gram or ops.h_gram, combine or ops.h_combine
    return gram, combine


def _as_numpy(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def pca_step(x, K, gram=None, combine=None):
    """the top K principal directions of the rows of x ([n][d] fp32): (V fp64 [K][d] unit rows before any sign fix,
    λ fp64 [K] the Gram eigenvalues, largest first, trace G).  gram / combine: ops.h_gram / ops.h_combine, or
    stand-ins with their contract (oracle/hspace.py restates them in numpy)."""
    gram, combine = _kernels(gram, combine)
    n = x.shape[0]
    if not 1 <= K <= n - 1:
        raise ValueError(f"K={K} principal components need at least K + 1 = {K + 1} samples, got {n}")
    like = (lambda a: torch.as_tensor(a, device=x.device)) if torch.is_tensor(x) else np.asarray
    mu = combine(x, like(np.full((1, n), 1.0 / n)))[0]
    G = _as_numpy(gram(x, mu))
    lam, U = np.linalg.eigh(G)
    order = np.argsort(lam, kind="stable")[::-1][:K]
    lam, U = lam[order], U[:, order]
    # a component at the rounding level of the largest is not a direction of the data: 1 / sqrt(λ) would amplify noise
    ok = lam > 1e-10 * max(float(lam[0]), 0.0)
    if not (lam[0] > 0 and ok.all()):
        bad = int(np.argmin(ok)) if lam[0] > 0 else 0
        raise ValueError(f"principal component {bad} has variance {lam[bad]:.3g}, at the rounding level of the "
                         f"largest ({lam[0]:.3g}): the samples span fewer than K={K} directions")
    V = _as_numpy(combine(x, like(np.ascontiguousarray((U / np.sqrt(lam)).T)), mu))
    return V, lam, float(np.trace(G))


def mean_diff_step(x, n_pos, combine=None):
    """(μ₊, μ₋) fp64 [d] of the first n_pos rows of x and of the others, one h_combine of two weight rows (1/n on the
    set's rows, 0 on the other's): a set compared with itself gives the same bits twice"""
    combine = _kernels(None, combine)[1]
    n = x.shape[0]
    if not 1 <= n_pos < n:
        raise ValueError(f"mean difference: {n_pos} positive and {n - n_pos} negative samples; each set needs one")
    w = np.zeros((2, n))
    w[0, :n_pos] = 1.0 / n_pos
    w[1, n_pos:] = 1.0 / (n - n_pos)
    like = (lambda a: torch.as_tensor(a, device=x.device)) if torch.is_tensor(x) else np.asarray
    m = _as_numpy(combine(x, like(w)))
    return m[0], m[1]


def fix_signs(V, prev=None):
    """V [K][d] with each row's sign fixed: without prev (the first step) its largest-|value| entry (the first one on
    a tie) positive, else its dot product with prev's row >= 0"""
    V = np.array(V, dtype=np.float64, copy=True)
    for k in range(V.shape[0]):
        if prev is None:
            flip = V[k, int(np.argmax(np.abs(V[k])))] < 0
        else:
            flip = float(np.dot(V[k], prev[k])) < 0
        if flip:
            V[k] = -V[k]
    return V


def _cos(a, b):
    na, nb = float(np.linalg.norm(a)), float(np.linalg.norm(b))
    return float(np.dot(a, b)) / (na * nb) if na > 0 and nb > 0 else float("nan")


def discover(X, ts, K=None, n_pos=None, gram=None, combine=None):
    """directions of every step: X [steps][n][d] fp32 (step k at timestep ts[k], largest t first); K for PCA, n_pos
    (the first n_pos rows positive) for the mean difference.  Returns (directions, tsv rows): directions is a list of
    (kind, component, {t: fp64 [d]}, {t: (variance, ratio)} | None); a tsv row is (t, values...)."""
    if (K is None) == (n_pos is None):
        raise ValueError("discover: give K (PCA) or n_pos (mean difference)")
    steps, n = X.shape[0], X.shape[1]
    rows = []
    if K is not None:
        dirs = [{} for _ in range(K)]
        ev = [{} for _ in range(K)]
        prev = None
        for k in range(steps):
            V, lam, tr = pca_step(X[k], K, gram, combine)
            V = fix_signs(V, prev)
            t = int(ts[k])
            row = [t]
            for c in range(K):
                var = float(lam[c]) / (n - 1)
                dirs[c][t] = V[c] * math.sqrt(var)
                ev[c][t] = (var, float(lam[c]) / tr)
                row += [var, float(lam[c]) / tr, _cos(V[c], prev[c]) if prev is not None else float("nan")]
            rows.append(tuple(row))
            prev = V
        return [("pca", c, dirs[c], ev[c]) for c in range(K)], rows
    d = {}
    for k in range(steps):
        mp, mn = mean_diff_step(X[k], n_pos, combine)
        t = int(ts[k])
        d[t] = mp - mn
        rows.append((t, float(np.linalg.norm(d[t])), float(np.linalg.norm(mp)), float(np.linalg.norm(mn))))
    return [("mean_diff", 0, d, None)], rows


def tsv_text(kind, rows, K=1):
    """h_directions.tsv: one row per timestep"""
    if kind == "pca":
        head = ["t"] + [f"pc{c}_{s}" for c in range(K) for s in ("variance", "ratio", "cos_prev")]
    else:
        head = ["t", "norm_d", "norm_mu_pos", "norm_mu_neg"]
    lines = ["\t".join(head)]
    for r in rows:
        lines.append("\t".join([str(int(r[0]))] + [f"{float(v):.9g}" for v in r[1:]]))
    return "\n".join(lines) + "\n"


def file_name(kind, component):
    return f"pc{component}.pth" if kind == "pca" else "mean_diff.pth"


def direction_dict(kind, component, delta_h, ev, shape, meta):
    """the torch.save dict of one direction: meta holds category, mid_ch, t_0, n_test_step and n"""
    out = {"format": FORMAT, "kind": kind, "component": int(component), **meta,
           "delta_h": {int(t): torch.from_numpy(np.asarray(v, dtype=np.float32).reshape(shape)) for t, v in
                       delta_h.items()}}
    if ev is not None:
        out["explained_variance"] = {int(t): (float(a), float(b)) for t, (a, b) in ev.items()}
    return out


def write_directions(out_dir, directions, rows, shape, meta):
    """pc<k>.pth / mean_diff.pth and h_directions.tsv under out_dir; returns the paths of the direction files"""
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for kind, comp, dh, ev in directions:
        p = os.path.join(out_dir, file_name(kind, comp))
        torch.save(direction_dict(kind, comp, dh, ev, shape, meta), p)
        paths.append(p)
    with open(os.path.join(out_dir, "h_directions.tsv"), "w") as f:
        f.write(tsv_text(directions[0][0], rows, len(directions)))
    return paths


def load_direction(path, config, args, mid_ch):
    """a direction file checked against the run: ValueError naming the field when its format tag, category, mid_ch
    (the model's bottleneck channels), t_0 or n_test_step differ from the run's"""
    obj = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(obj, dict) or obj.get("format") != FORMAT:
        got = obj.get("format") if isinstance(obj, dict) else type(obj).__name__
        raise ValueError(f"{path}: field 'format' is {got!r}, not {FORMAT!r}: not an h-space direction file "
                         "(raw Δh dicts and DeltaBlock checkpoints load through --train_delta_h / the checkpoint name)")
    for field, want in (("category", config.data.category), ("mid_ch", int(mid_ch)), ("t_0", int(args.t_0)),
                        ("n_test_step", int(args.n_test_step))):
        if obj.get(field) != want:
            raise ValueError(f"{path}: field {field!r} is {obj.get(field)!r}, this run has {want!r}")
    return obj


def direction_rows(obj, edit_ts):
    """fp32 [n_edit][C][h][w]: the direction at every edit timestep; KeyError naming a timestep with no entry"""
    rows = []
    for t in edit_ts:
        if int(t) not in obj["delta_h"]:
            raise KeyError(f"the direction file has no entry for edit timestep t={int(t)} (it holds "
                           f"{sorted(obj['delta_h'])[:3]}..)")
        rows.append(obj["delta_h"][int(t)].float())
    return torch.stack(rows) if rows else None
