"""numpy fp64 restatement of h-space direction discovery (asyrp_official_b200/hspace.py).

PCA here goes through the SVD of the centred data, an independent route from the engine's Gram + eigh + projection;
gram / combine restate the two statistics kernels (csrc/hspace.cu) for comparisons and host-side runs.
"""
import numpy as np


def gram(x, mu):
    """G[i][j] = sum_k (x[i][k] - mu[k]) (x[j][k] - mu[k])"""
    xc = np.asarray(x, np.float64) - np.asarray(mu, np.float64)[None]
    return xc @ xc.T


def combine(x, w, mu=None):
    """out[k][j] = sum_r w[k][r] (x[r][j] - mu[j]), the rows r in order from 0 as the kernel adds them"""
    xc = np.asarray(x, np.float64)
    if mu is not None:
        xc = xc - np.asarray(mu, np.float64)[None]
    w = np.asarray(w, np.float64)
    out = np.zeros((w.shape[0], xc.shape[1]))
    for r in range(xc.shape[0]):
        out += w[:, r:r + 1] * xc[r][None]
    return out


def sign_rule(V, prev=None):
    """first step: each row's largest-|value| entry positive; later steps: dot with the previous step's row >= 0"""
    V = np.array(V, np.float64)
    for k in range(V.shape[0]):
        ref = V[k, np.argmax(np.abs(V[k]))] if prev is None else V[k] @ prev[k]
        if ref < 0:
            V[k] *= -1
    return V


def pca(X, K):
    """X [steps][n][d]: per step (unit components [K][d] with the sign rule applied, variances λ / (n - 1) [K], ratios
    λ / sum of all λ [K], stored directions [K][d] = unit * sqrt(λ / (n - 1)))"""
    out, prev = [], None
    for x in np.asarray(X, np.float64):
        n = x.shape[0]
        xc = x - x.mean(axis=0)
        _, S, Vt = np.linalg.svd(xc, full_matrices=False)
        lam = S[:K] ** 2
        V = sign_rule(Vt[:K], prev)
        var = lam / (n - 1)
        out.append((V, var, lam / np.sum(S ** 2), V * np.sqrt(var)[:, None]))
        prev = V
    return out


def mean_diff(X, n_pos):
    """X [steps][n][d], the first n_pos rows positive: per step (μ₊ - μ₋, |μ₊ - μ₋|, |μ₊|, |μ₋|)"""
    out = []
    for x in np.asarray(X, np.float64):
        mp, mn = x[:n_pos].mean(axis=0), x[n_pos:].mean(axis=0)
        d = mp - mn
        out.append((d, np.linalg.norm(d), np.linalg.norm(mp), np.linalg.norm(mn)))
    return out


def tsv(kind, ts, per_step):
    """h_directions.tsv from pca() / mean_diff() results"""
    if kind == "pca":
        K = per_step[0][0].shape[0]
        lines = ["\t".join(["t"] + [f"pc{c}_{s}" for c in range(K) for s in ("variance", "ratio", "cos_prev")])]
        for k, (V, var, ratio, _) in enumerate(per_step):
            cells = [str(int(ts[k]))]
            for c in range(K):
                cos = float("nan") if k == 0 else float(V[c] @ per_step[k - 1][0][c]) / (
                    np.linalg.norm(V[c]) * np.linalg.norm(per_step[k - 1][0][c]))
                cells += [f"{float(var[c]):.9g}", f"{float(ratio[c]):.9g}", f"{cos:.9g}"]
            lines.append("\t".join(cells))
    else:
        lines = ["t\tnorm_d\tnorm_mu_pos\tnorm_mu_neg"]
        for k, (_, nd, npos, nneg) in enumerate(per_step):
            lines.append("\t".join([str(int(ts[k]))] + [f"{float(v):.9g}" for v in (nd, npos, nneg)]))
    return "\n".join(lines) + "\n"
