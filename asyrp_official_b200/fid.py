"""Inception-v3 pool features on the engine's kernels, and the FID and KID that `--fid` reports for each set of edits.

The reference has no realism score: the network and the metric here are this project's definition, following
pytorch-fid (FID) and torch-fidelity (KID).  The network is pytorch-fid's FID Inception-v3, whose weights file is
pt_inception-2015-12-05-6726825d.pth (a state dict with torchvision Inception3 key names), evaluated up to the 2048-d
global average pool:

    input      the image its PNG shows, then what pytorch-fid does to a PNG: u8 = clamp((x + 1) * 0.5 * 255 + 0.5, 0,
               255) truncated (torchvision's save_image), / 255, bilinear resize to 299 x 299 (align_corners=False),
               2 v - 1
    stem       Conv2d_1a_3x3 (/2), 2a_3x3, 2b_3x3 (pad 1), max-pool 3x3 / 2, 3b_1x1, 4a_3x3, max-pool 3x3 / 2
    Mixed_5b-d FIDInceptionA (pool features 32, 64, 64)        branch_pool: avg-pool 3x3 / 1 pad 1, count_include_pad
    Mixed_6a   InceptionB                                                   False, then a 1x1 BasicConv2d
    Mixed_6b-e FIDInceptionC (c7 = 128, 160, 160, 192)          the same avg-pool
    Mixed_7a   InceptionD
    Mixed_7b   FIDInceptionE_1                                  the same avg-pool
    Mixed_7c   FIDInceptionE_2                                  max-pool 3x3 / 1 pad 1 (padding never wins the max)
    features   mean over the 8 x 8 pixels -> 2048; fc is not evaluated

BasicConv2d is conv (no bias) -> BN (eps 1e-3) -> ReLU; the BN is folded into the conv's weight and bias at load time
(exact algebra, fp64 on the host).  Every conv is the TF32 implicit GEMM of csrc/tf32_gemm.cuh writing its channel
slice of the block output, so no concatenation is materialised; a branch narrower than a multiple of 64 channels runs
with zero weight rows and stores only its own channels.

Sets: every hs_coeff tuple of a run (each --delta_interpolation strength, each --multiple_attr tuple, each --attr_sweep
attribute) is one edited set, scored against the origin DDIM pass of the same x_T; train and test passes are separate.

    FID  = |mu1 - mu2|^2 + tr S1 + tr S2 - 2 sum_i sqrt(l_i), l the eigenvalues (clamped at 0) of S1^1/2 S2 S1^1/2, mu
           and S (n - 1 denominator, as np.cov) in fp64.  This is tr sqrtm(S1 S2) for PSD matrices, and unlike
           scipy.linalg.sqrtm it is well defined when n < 2048 makes S rank-deficient.
    KID  = the unbiased MMD^2 with k(x, y) = (x . y / 2048 + 1)^3 over all rows of both sets, the diagonal excluded in
           the two within-set sums: torch-fidelity's KID mean with kid_subset_size = n.

A set of fewer than two images gets nan for both.  The moments and the kernel sums run on the GPU in fp64
(csrc/fid.cu); the two 2048^2 eigendecompositions per set run on the host in fp64.

Real images (--fid_ref STATS.npz): `python -m asyrp_official_b200.fid --save-stats DIR OUT.npz --fid_weights W` reads
every image directly in DIR as pytorch-fid does (Image.open(p).convert('RGB') at its own size: no resize or crop to
the edits' size), runs the u8 through features_u8 (pytorch-fid's ToTensor path, the same bits as features of
u8 / 127.5 - 1) and writes mu / sigma (pytorch-fid's keys, fp64), the features (fp32) and kid_kxx (their kernel sum
without the diagonal).  A run then scores its origin set and each edited set against that file:

    FID       as above against the file's mu / sigma (a pytorch-fid --save-stats file works too)
    KID       the full-set KID, the reference's within-set sum taken from kid_kxx
    KID_mean  torch-fidelity's KID mean / std over random subsets (kid_subsets: kid_subsets subsets of
    KID_std   kid_subset_size rows, RandomState(2020), the edited set drawn first); nan when a set is smaller

The KID columns are nan for a file without features.

Precision / recall / density / coverage (--prdc, prdc): improved precision / recall (Kynkaanniemi et al. 2019) and
density / coverage (Naeem et al. 2020, the prdc package) from k-nearest-neighbour balls of the same pool features, on
squared distances in fp64 (csrc/prdc.cu); real = the origin set, or the file's features with --fid_ref.  With k = 3,
precision and recall are those of guided-diffusion's ADM evaluator except that it counts ties (<=) and computes its
distances in fp16 (fp32 fallback); here every comparison is strict and every distance fp64.  The Inception score is
not computed.

No real pt_inception-2015-12-05-6726825d.pth has been loaded by this project's tests: the key list below follows
torchvision's Inception3, and the loader refuses any other layout by name.
"""
import argparse
import math
import os
import sys
import time
import warnings

import numpy as np
import torch

from . import _lib, ops

BN_EPS = 1e-3
SIZE = 299
DIMS = 2048
BN_STATS = ("weight", "bias", "running_mean", "running_var")
FC = {"fc.weight": (1008, DIMS), "fc.bias": (1008,)}  # the logits layer: accepted, checked and ignored
# fp32 bytes of the activations live at once per image at the peak (the stem's Conv2d_2b: the packed input, 2a's
# output and 2b's): rows run in chunks of ACTIVATION_BUDGET // ROW_BYTES images
ROW_BYTES = 4 * (SIZE * SIZE * 4 + 147 * 147 * (32 + 64))
ACTIVATION_BUDGET = 1 << 30

# name -> (cin, cout, kh, kw, stride, pad_h, pad_w) of the stem's BasicConv2d layers
STEM = {"Conv2d_1a_3x3": (3, 32, 3, 3, 2, 0, 0), "Conv2d_2a_3x3": (32, 32, 3, 3, 1, 0, 0),
        "Conv2d_2b_3x3": (32, 64, 3, 3, 1, 1, 1), "Conv2d_3b_1x1": (64, 80, 1, 1, 1, 0, 0),
        "Conv2d_4a_3x3": (80, 192, 3, 3, 1, 0, 0)}
# (block, kind, in channels, pool features / c7)
BLOCKS = (("Mixed_5b", "A", 192, 32), ("Mixed_5c", "A", 256, 64), ("Mixed_5d", "A", 288, 64),
          ("Mixed_6a", "B", 288, None), ("Mixed_6b", "C", 768, 128), ("Mixed_6c", "C", 768, 160),
          ("Mixed_6d", "C", 768, 160), ("Mixed_6e", "C", 768, 192), ("Mixed_7a", "D", 768, None),
          ("Mixed_7b", "E1", 1280, None), ("Mixed_7c", "E2", 2048, None))
# the branches of a block in output-channel order: (pool before the first conv or None, [conv, ...]); the last entry
# of a branch writes the block output, a pair of convs both reading the previous one writes two adjacent slices, a
# branch without convs is the pool alone
BRANCHES = {
    "A": ((None, ["branch1x1"]), (None, ["branch5x5_1", "branch5x5_2"]),
          (None, ["branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"]), ("avg", ["branch_pool"])),
    "B": ((None, ["branch3x3"]), (None, ["branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"]), ("max2", [])),
    "C": ((None, ["branch1x1"]), (None, ["branch7x7_1", "branch7x7_2", "branch7x7_3"]),
          (None, ["branch7x7dbl_1", "branch7x7dbl_2", "branch7x7dbl_3", "branch7x7dbl_4", "branch7x7dbl_5"]),
          ("avg", ["branch_pool"])),
    "D": ((None, ["branch3x3_1", "branch3x3_2"]),
          (None, ["branch7x7x3_1", "branch7x7x3_2", "branch7x7x3_3", "branch7x7x3_4"]), ("max2", [])),
    "E1": ((None, ["branch1x1"]), (None, ["branch3x3_1", ("branch3x3_2a", "branch3x3_2b")]),
           (None, ["branch3x3dbl_1", "branch3x3dbl_2", ("branch3x3dbl_3a", "branch3x3dbl_3b")]),
           ("avg", ["branch_pool"])),
}
BRANCHES["E2"] = BRANCHES["E1"][:3] + (("max1", ["branch_pool"]),)
POOL_MODE = {"avg": ops.FID_POOL_AVG3S1, "max1": ops.FID_POOL_MAX3S1, "max2": ops.FID_POOL_MAX3S2}


def block_convs(kind, cin, arg):
    """conv name -> (cin, cout, kh, kw, stride, pad_h, pad_w) of one block (torchvision's Inception A-E layers)"""
    if kind == "A":
        return {"branch1x1": (cin, 64, 1, 1, 1, 0, 0), "branch5x5_1": (cin, 48, 1, 1, 1, 0, 0),
                "branch5x5_2": (48, 64, 5, 5, 1, 2, 2), "branch3x3dbl_1": (cin, 64, 1, 1, 1, 0, 0),
                "branch3x3dbl_2": (64, 96, 3, 3, 1, 1, 1), "branch3x3dbl_3": (96, 96, 3, 3, 1, 1, 1),
                "branch_pool": (cin, arg, 1, 1, 1, 0, 0)}
    if kind == "B":
        return {"branch3x3": (cin, 384, 3, 3, 2, 0, 0), "branch3x3dbl_1": (cin, 64, 1, 1, 1, 0, 0),
                "branch3x3dbl_2": (64, 96, 3, 3, 1, 1, 1), "branch3x3dbl_3": (96, 96, 3, 3, 2, 0, 0)}
    if kind == "C":
        c7 = arg
        return {"branch1x1": (cin, 192, 1, 1, 1, 0, 0), "branch7x7_1": (cin, c7, 1, 1, 1, 0, 0),
                "branch7x7_2": (c7, c7, 1, 7, 1, 0, 3), "branch7x7_3": (c7, 192, 7, 1, 1, 3, 0),
                "branch7x7dbl_1": (cin, c7, 1, 1, 1, 0, 0), "branch7x7dbl_2": (c7, c7, 7, 1, 1, 3, 0),
                "branch7x7dbl_3": (c7, c7, 1, 7, 1, 0, 3), "branch7x7dbl_4": (c7, c7, 7, 1, 1, 3, 0),
                "branch7x7dbl_5": (c7, 192, 1, 7, 1, 0, 3), "branch_pool": (cin, 192, 1, 1, 1, 0, 0)}
    if kind == "D":
        return {"branch3x3_1": (cin, 192, 1, 1, 1, 0, 0), "branch3x3_2": (192, 320, 3, 3, 2, 0, 0),
                "branch7x7x3_1": (cin, 192, 1, 1, 1, 0, 0), "branch7x7x3_2": (192, 192, 1, 7, 1, 0, 3),
                "branch7x7x3_3": (192, 192, 7, 1, 1, 3, 0), "branch7x7x3_4": (192, 192, 3, 3, 2, 0, 0)}
    return {"branch1x1": (cin, 320, 1, 1, 1, 0, 0), "branch3x3_1": (cin, 384, 1, 1, 1, 0, 0),
            "branch3x3_2a": (384, 384, 1, 3, 1, 0, 1), "branch3x3_2b": (384, 384, 3, 1, 1, 1, 0),
            "branch3x3dbl_1": (cin, 448, 1, 1, 1, 0, 0), "branch3x3dbl_2": (448, 384, 3, 3, 1, 1, 1),
            "branch3x3dbl_3a": (384, 384, 1, 3, 1, 0, 1), "branch3x3dbl_3b": (384, 384, 3, 1, 1, 1, 0),
            "branch_pool": (cin, 192, 1, 1, 1, 0, 0)}


def block_width(kind, cin, arg):
    """output channels of a block: the widths of its branches' last convs, plus cin for a pool-only branch"""
    return {"A": 224 + (arg or 0), "B": 480 + cin, "C": 768, "D": 512 + cin}.get(kind, 2048)


def conv_specs():
    """full conv name (e.g. 'Mixed_6b.branch7x7_2') -> (cin, cout, kh, kw, stride, pad_h, pad_w), in network order"""
    out = dict(STEM)
    for name, kind, cin, arg in BLOCKS:
        out.update({f"{name}.{k}": v for k, v in block_convs(kind, cin, arg).items()})
    return out


def state_dict_shapes():
    """name -> shape of every tensor the network evaluates (without fc and num_batches_tracked)"""
    shapes = {}
    for name, (cin, cout, kh, kw, *_) in conv_specs().items():
        shapes[f"{name}.conv.weight"] = (cout, cin, kh, kw)
        for s in BN_STATS:
            shapes[f"{name}.bn.{s}"] = (cout,)
    return shapes


def load_state_dict(sd_or_path):
    """Validate an FID Inception-v3 state dict (or the path of its torch.save) and return the tensors the network
    evaluates as fp32 on the host, keyed as in the state dict.  fc.weight / fc.bias and every BN's num_batches_tracked
    are accepted and ignored.  Raises ValueError naming the key on a missing, mis-shaped or unknown key, and on a file
    that is not a state dict."""
    sd = sd_or_path
    if not isinstance(sd, dict):
        try:
            sd = torch.load(sd_or_path, map_location="cpu", weights_only=True)
        except Exception as e:  # a truncated file, another format, ...
            raise ValueError(f"FID Inception weights {sd_or_path!r}: cannot be read as a torch.save'd state dict "
                             f"({e})") from None
        if not isinstance(sd, dict):
            raise ValueError(f"FID Inception weights {sd_or_path!r}: not a state dict (got {type(sd).__name__})")
    expected = state_dict_shapes()
    tracked = {f"{n}.bn.num_batches_tracked" for n in conv_specs()}
    unknown = sorted(k for k in sd if k not in expected and k not in FC and k not in tracked)
    if unknown:
        raise ValueError(f"FID Inception state dict: unexpected keys {unknown[:8]}{' ...' if len(unknown) > 8 else ''} "
                         "(expected the layout of pytorch-fid's FID Inception-v3)")
    for k, shape in FC.items():
        if k in sd and tuple(torch.as_tensor(sd[k]).shape) != shape:
            raise ValueError(f"FID Inception state dict: {k!r} has shape {tuple(torch.as_tensor(sd[k]).shape)}, "
                             f"expected {shape}")
    out = {}
    for k, shape in expected.items():
        if k not in sd:
            raise ValueError(f"FID Inception state dict: missing key {k!r}")
        t = torch.as_tensor(sd[k])
        if tuple(t.shape) != shape:
            raise ValueError(f"FID Inception state dict: {k!r} has shape {tuple(t.shape)}, expected {shape}")
        out[k] = t.detach().float().cpu().contiguous()
    return out


def fold(sd):
    """conv name -> (weight [cout][cin][kh][kw], bias [cout]) fp32 of a load_state_dict() result: the BN (eps 1e-3)
    folded into the bias-free conv in fp64, w' = w * g / sqrt(var + eps), b' = beta - mean * g / sqrt(var + eps)"""
    out = {}
    for name in conv_specs():
        g = {s: sd[f"{name}.bn.{s}"].double() for s in BN_STATS}
        scale = g["weight"] / torch.sqrt(g["running_var"] + BN_EPS)
        w = sd[f"{name}.conv.weight"].double() * scale[:, None, None, None]
        out[name] = (w.float().contiguous(), (g["bias"] - g["running_mean"] * scale).float().contiguous())
    return out


def frechet_distance(mu1, sigma1, mu2, sigma2):
    """|mu1 - mu2|^2 + tr S1 + tr S2 - 2 sum sqrt(eig(S1^1/2 S2 S1^1/2)), eigenvalues clamped at 0; fp64 on the host"""
    mu1, mu2 = (np.asarray(m, dtype=np.float64) for m in (mu1, mu2))
    s1, s2 = (np.asarray(s, dtype=np.float64) for s in (sigma1, sigma2))
    lam, vec = np.linalg.eigh((s1 + s1.T) / 2)
    root = (vec * np.sqrt(np.clip(lam, 0, None))) @ vec.T
    m = root @ s2 @ root
    ev = np.clip(np.linalg.eigvalsh((m + m.T) / 2), 0, None)
    diff = mu1 - mu2
    return float(diff @ diff + np.trace(s1) + np.trace(s2) - 2 * np.sqrt(ev).sum())


def kid_from_sums(kxx, kyy, kxy, n, m):
    """the unbiased MMD^2 from the kernel sums: kxx, kyy without their diagonals, kxy over all n * m pairs"""
    return kxx / (n * (n - 1)) + kyy / (m * (m - 1)) - 2 * kxy / (n * m)


def kid(f1, f2):
    """KID of two feature sets fp32 [n][d] / [m][d] on the device (n, m >= 2): kernel sums on the GPU in fp64"""
    n, m = f1.shape[0], f2.shape[0]
    kxx = ops.fid_kernel_sum(f1, f1, exclude_diag=True).item()
    kyy = ops.fid_kernel_sum(f2, f2, exclude_diag=True).item()
    kxy = ops.fid_kernel_sum(f1, f2).item()
    return kid_from_sums(kxx, kyy, kxy, n, m)


def set_moments(f):
    """(mu, sigma) of a feature set fp32 [n][d] on the device, fp64 numpy on the host"""
    mu, sigma = ops.fid_moments(f.contiguous())
    return mu.cpu().numpy(), sigma.cpu().numpy()


def fid_kid(ref, edited, ref_moments=None):
    """(FID, KID) of the feature sets ref and edited (fp32 [n][d] on the device, rows in image order); nan for both when
    either set has fewer than two rows.  ref_moments: set_moments(ref), when several sets share the reference."""
    if ref.shape[0] < 2 or edited.shape[0] < 2:
        print(f"FID / KID: a set of {min(ref.shape[0], edited.shape[0])} image(s) has no covariance: nan")
        return math.nan, math.nan
    mu1, s1 = ref_moments if ref_moments is not None else set_moments(ref)
    mu2, s2 = set_moments(edited)
    return frechet_distance(mu1, s1, mu2, s2), kid(ref.contiguous(), edited.contiguous())


def kid_subset_indices(n, m, subsets, size, seed=2020):
    """int32 [subsets][size] row indices into the scored set (n rows) and the reference (m rows): a fresh
    RandomState(seed), per subset in order choice(n, size, replace=False) then choice(m, size, replace=False)"""
    rng = np.random.RandomState(seed)
    i1, i2 = np.empty((subsets, size), np.int32), np.empty((subsets, size), np.int32)
    for z in range(subsets):
        i1[z] = rng.choice(n, size, replace=False)
        i2[z] = rng.choice(m, size, replace=False)
    return i1, i2


def kid_subsets(f1, f2, subsets, size, seed=2020):
    """(mean, std) of the KID over random subsets, torch-fidelity's kid_features_to_metric: f1 the set scored, f2 the
    reference (fp32 [n][d] / [m][d] on the device).  A fresh np.random.RandomState(seed) draws, for each subset in
    order, size rows of f1 and then size rows of f2 without replacement; each subset's MMD^2 is kid_from_sums of its
    three kernel sums (the diagonal excluded within a set); np.mean and np.std (ddof 0) of the subsets' values.  The
    sums of all subsets run in three launches.  (nan, nan) and a printed warning when a set has fewer than size rows
    (torch-fidelity raises there)."""
    if subsets < 1 or size < 2:
        raise ValueError(f"kid_subsets: needs subsets >= 1 and size >= 2, got {subsets} and {size}")
    n, m = f1.shape[0], f2.shape[0]
    if n < size or m < size:
        print(f"KID subsets: a set of {min(n, m)} rows is smaller than the subset size {size}: nan")
        return math.nan, math.nan
    i1, i2 = kid_subset_indices(n, m, subsets, size, seed)
    t1, t2 = torch.from_numpy(i1).to(f1.device), torch.from_numpy(i2).to(f1.device)
    f1, f2 = f1.contiguous(), f2.contiguous()
    kxx = ops.fid_kernel_sum_subsets(f1, f1, t1, t1, exclude_diag=True).cpu().numpy()
    kyy = ops.fid_kernel_sum_subsets(f2, f2, t2, t2, exclude_diag=True).cpu().numpy()
    kxy = ops.fid_kernel_sum_subsets(f1, f2, t1, t2).cpu().numpy()
    mmd = kid_from_sums(kxx, kyy, kxy, size, size)
    return float(np.mean(mmd)), float(np.std(mmd))


def score_against_stats(f, real, subsets, size, moments=None):
    """(FID, KID, KID_mean, KID_std) of the feature set f (fp32 [n][d] on the device) against reference statistics
    real (load_stats, its features moved to the device): FID against mu / sigma; the full-set KID from real's kid_kxx
    and f's two kernel sums; the subset KID (kid_subsets, f first) when subsets > 0.  The KID values are nan without
    features in real, all four are nan when f has fewer than two rows.  moments: set_moments(f) when already known."""
    n = f.shape[0]
    if n < 2:
        print(f"FID / KID against the real images: a set of {n} image(s) has no covariance: nan")
        return math.nan, math.nan, math.nan, math.nan
    mu, sigma = moments if moments is not None else set_moments(f)
    fd = frechet_distance(mu, sigma, real["mu"], real["sigma"])
    if "features" not in real:
        return fd, math.nan, math.nan, math.nan
    ref = real["features"]
    kxx = ops.fid_kernel_sum(f, f, exclude_diag=True).item()
    kxy = ops.fid_kernel_sum(f, ref).item()
    kd = kid_from_sums(kxx, real["kid_kxx"], kxy, n, ref.shape[0])
    km, ks = kid_subsets(f, ref, subsets, size) if subsets > 0 else (math.nan, math.nan)
    return fd, kd, km, ks


# ---- precision / recall / density / coverage (--prdc) from k-nearest-neighbour balls ----
def knn_radii(f, k):
    """fp64 [n] on the device: the squared distance of each row of the feature set f (fp32 [n][d] on the device) to its
    k-th nearest other row, duplicates counted: the (k + 1)-th smallest D(f_i, f_j) over every j, j = i included
    (prdc's compute_nearest_neighbour_distances, squared).  1 <= k <= 32 and n > k."""
    return ops.fid_knn_radii(f.contiguous(), int(k))


def prdc(real, fake, k, real_radii=None):
    """(precision, recall, density, coverage) as floats (fp64) of the fake set against the real set (fp32 [n][d] /
    [m][d] on the device), prdc.compute_prdc's definitions on squared distances with strict <:
        precision = #{j : some i has D(r_i, f_j) < r_k(i)} / m
        recall    = #{i : some j has D(r_i, f_j) < r_k^fake(j)} / n
        density   = #{(i, j) : D(r_i, f_j) < r_k(i)} / (k m)
        coverage  = #{i : some j has D(r_i, f_j) < r_k(i)} / n
    r_k the knn_radii of the real set (real_radii, when several fake sets share it) and r_k^fake those of the fake set.
    All four are nan, with a warning, when either set has k rows or fewer."""
    n, m = real.shape[0], fake.shape[0]
    if n <= k or m <= k:
        warnings.warn(f"precision / recall / density / coverage: a set of {min(n, m)} rows has no {k}-th nearest "
                      "neighbour: nan", RuntimeWarning, stacklevel=2)
        return math.nan, math.nan, math.nan, math.nan
    real, fake = real.contiguous(), fake.contiguous()
    rr = real_radii if real_radii is not None else knn_radii(real, k)
    b_in_a, a_in_b, a_covered = ops.fid_knn_counts(real, rr, fake, knn_radii(fake, k))
    counts = torch.stack([(b_in_a > 0).sum(), (a_in_b > 0).sum(), b_in_a.sum(), (a_covered > 0).sum()]).tolist()
    return counts[0] / m, counts[1] / n, counts[2] / (k * m), counts[3] / n


# ---- reference statistics (.npz): pytorch-fid's keys mu / sigma, plus this project's features / kid_kxx for KID ----
# key -> (dtype, shape); None: any length >= 2
STATS_KEYS = {"mu": (np.float64, (DIMS,)), "sigma": (np.float64, (DIMS, DIMS)), "features": (np.float32, (None, DIMS)),
              "kid_kxx": (np.float64, ())}
SAVE_STATS_HINT = "make one with python -m asyrp_official_b200.fid --save-stats DIR OUT.npz --fid_weights W"


def validate_stats(path):
    """Check a reference statistics file's keys, dtypes and shapes from the .npy headers alone (no array is read).
    Returns (number of reference rows or None, whether it holds features / kid_kxx for KID).  mu / sigma are required;
    features and kid_kxx come together.  Raises ValueError naming the key or the problem."""
    import zipfile
    what = f"FID reference statistics {path!r}"
    if os.path.isdir(path):
        raise ValueError(f"{what} is a directory, not a statistics file: {SAVE_STATS_HINT}")
    if not os.path.isfile(path):
        raise ValueError(f"{what}: no such file ({SAVE_STATS_HINT})")
    if not zipfile.is_zipfile(path):
        raise ValueError(f"{what}: not an .npz file")
    headers = {}
    try:
        with zipfile.ZipFile(path) as zf:
            for name in zf.namelist():
                key = name[:-4] if name.endswith(".npy") else name
                with zf.open(name) as f:
                    version = np.lib.format.read_magic(f)
                    read = {(1, 0): np.lib.format.read_array_header_1_0,
                            (2, 0): np.lib.format.read_array_header_2_0}.get(version)
                    if read is None:
                        raise ValueError(f"{key!r} has .npy format version {version}")
                    shape, _, dtype = read(f)
                headers[key] = (dtype, tuple(shape))
    except (zipfile.BadZipFile, OSError, EOFError, ValueError) as e:
        raise ValueError(f"{what}: cannot be read ({e})") from None
    unknown = sorted(set(headers) - set(STATS_KEYS))
    if unknown:
        raise ValueError(f"{what}: unexpected keys {unknown} (expected mu, sigma and optionally features, kid_kxx)")
    for key in ("mu", "sigma"):
        if key not in headers:
            raise ValueError(f"{what}: missing key {key!r}")
    if ("features" in headers) != ("kid_kxx" in headers):
        missing = "kid_kxx" if "features" in headers else "features"
        raise ValueError(f"{what}: missing key {missing!r} (features and kid_kxx come together)")
    for key, (dtype, shape) in headers.items():
        want_dtype, want_shape = STATS_KEYS[key]
        if dtype != np.dtype(want_dtype):
            raise ValueError(f"{what}: {key!r} has dtype {dtype}, expected {np.dtype(want_dtype)}")
        if len(shape) != len(want_shape) or any(w is not None and s != w for s, w in zip(shape, want_shape)) or \
                (key == "features" and shape[0] < 2):
            raise ValueError(f"{what}: {key!r} has shape {shape}, expected "
                             f"{tuple('N >= 2' if w is None else w for w in want_shape)}")
    has_features = "features" in headers
    return (headers["features"][1][0] if has_features else None), has_features


def load_stats(path, with_features=True):
    """the validated statistics of path: {'mu', 'sigma'} fp64 numpy, plus 'features' fp32 [N][2048] and 'kid_kxx'
    (float) when with_features and the file holds them"""
    _, has_features = validate_stats(path)
    with np.load(path, allow_pickle=False) as z:
        out = {"mu": z["mu"], "sigma": z["sigma"]}
        if with_features and has_features:
            out["features"] = z["features"]
            out["kid_kxx"] = float(z["kid_kxx"])
    return out


def stats_arrays(feats):
    """the arrays of a statistics file for the feature set feats fp32 [N][2048] on the device (N >= 2): mu and sigma
    (set_moments), the features and kid_kxx, their kernel sum without the diagonal (ops.fid_kernel_sum)"""
    feats = feats.contiguous()
    mu, sigma = set_moments(feats)
    kxx = ops.fid_kernel_sum(feats, feats, exclude_diag=True).cpu().numpy()
    return {"mu": mu, "sigma": sigma, "features": feats.cpu().numpy(), "kid_kxx": kxx}


def save_stats(path, feats):
    """write the statistics of feats (fp32 [N][2048] on the device, N >= 2) to path (write_stats)"""
    if feats.dim() != 2 or feats.shape[0] < 2 or feats.shape[1] != DIMS:
        raise ValueError(f"save_stats: needs features [N >= 2][{DIMS}], got {tuple(feats.shape)}")
    write_stats(path, stats_arrays(feats))


def write_stats(path, arrays):
    """arrays (key -> numpy array) as an uncompressed .npz that np.load reads (pytorch-fid reads its mu / sigma).  The
    members carry a fixed time stamp, so the same arrays give the same file bytes.  Written to a temporary file, then
    renamed."""
    import zipfile
    tmp = f"{path}.tmp.{os.getpid()}"
    with zipfile.ZipFile(tmp, "w", zipfile.ZIP_STORED, allowZip64=True) as zf:
        for key, a in arrays.items():
            with zf.open(zipfile.ZipInfo(f"{key}.npy", date_time=(1980, 1, 1, 0, 0, 0)), "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asarray(a, order="C"), allow_pickle=False)
    os.replace(tmp, path)


class FIDInception:
    """FIDInception(weights, device): features(x) -> fp32 [B][2048] on the device, the pool features of images
    x [B][3][H][W] in [-1, 1] (any size; quantised as their PNG, resized to 299 x 299).  Every operation is a kernel of
    libasyrp_b200.so; an image's features are bit-identical whatever batch it is in.  Rows run in chunks of max_rows
    images (default: ACTIVATION_BUDGET // ROW_BYTES), which bounds the activations at max_rows * ROW_BYTES bytes."""

    def __init__(self, state_dict_or_path, device=None, max_rows=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("FIDInception needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        folded = fold(load_state_dict(state_dict_or_path))
        self.max_rows = max(1, int(max_rows) if max_rows is not None else ACTIVATION_BUDGET // ROW_BYTES)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.specs = conv_specs()
        self.params = {}
        with torch.cuda.device(self.device):
            for name, (w, b) in folded.items():
                cout = w.shape[0]
                rows = -(-cout // 64) * 64  # the GEMM's 64-channel tiles: zero rows past the layer's width
                wp = torch.zeros(rows, *w.shape[1:])
                wp[:cout] = w
                bp = torch.zeros(rows)
                bp[:cout] = b
                packed = ops.pack_lpips_conv_weight(wp, cin_pad=4 if name == "Conv2d_1a_3x3" else None)
                self.params[name] = (packed.to(self.device), bp.to(self.device))

    def _conv(self, name, x, out=None):
        """BasicConv2d `name` of x into out (a new tensor, or a channel slice of the block output)"""
        _, cout, kh, kw, stride, ph, pw = self.specs[name]
        if out is None:
            B, H, W, _ = x.shape
            out = torch.empty(B, (H + 2 * ph - kh) // stride + 1, (W + 2 * pw - kw) // stride + 1, cout,
                              dtype=torch.float32, device=self.device)
        ops.fid_conv(x, *self.params[name], out, kh, kw, stride, (ph, pw), cstore=cout)
        return out

    def _block(self, name, kind, arg, x):
        B, H, W, cin = x.shape
        f32 = dict(dtype=torch.float32, device=self.device)
        Ho, Wo = ((H - 3) // 2 + 1, (W - 3) // 2 + 1) if kind in ("B", "D") else (H, W)
        out = torch.empty(B, Ho, Wo, block_width(kind, cin, arg), **f32)
        c0 = 0
        for pool, convs in BRANCHES[kind]:
            if not convs:  # the pool branch of InceptionB / D: the pooled input is the slice
                ops.fid_pool(x, out[..., c0:c0 + cin], POOL_MODE[pool])
                c0 += cin
                continue
            h = x
            if pool is not None:
                h = torch.empty(B, H, W, cin, **f32)
                ops.fid_pool(x, h, POOL_MODE[pool])
            for c in convs[:-1]:
                h = self._conv(f"{name}.{c}", h)
            for c in convs[-1] if isinstance(convs[-1], tuple) else (convs[-1],):
                cout = self.specs[f"{name}.{c}"][1]
                self._conv(f"{name}.{c}", h, out[..., c0:c0 + cout])
                c0 += cout
        return out

    def _maxpool(self, h):
        p = torch.empty(h.shape[0], (h.shape[1] - 3) // 2 + 1, (h.shape[2] - 3) // 2 + 1, h.shape[3],
                        dtype=torch.float32, device=self.device)
        ops.fid_pool(h, p, ops.FID_POOL_MAX3S2)
        return p

    def _chunk_features(self, x, u8=False):
        B = x.shape[0]
        f32 = dict(dtype=torch.float32, device=self.device)
        h = torch.empty(B, SIZE, SIZE, 4, **f32)
        if u8:
            ops.fid_pack_u8(x.to(self.device, non_blocking=True).contiguous(), h)
        else:
            ops.fid_pack(x.to(**f32).contiguous(), h)
        h = self._conv("Conv2d_2a_3x3", self._conv("Conv2d_1a_3x3", h))
        h = self._maxpool(self._conv("Conv2d_2b_3x3", h))
        h = self._maxpool(self._conv("Conv2d_4a_3x3", self._conv("Conv2d_3b_1x1", h)))
        for name, kind, _, arg in BLOCKS:
            h = self._block(name, kind, arg, h)
        feats = torch.empty(B, DIMS, **f32)
        ops.fid_mean(h, feats)
        return feats

    @torch.no_grad()
    def features(self, x):
        """pool features fp32 [B][2048] on the device"""
        x = torch.as_tensor(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] == 0:
            raise ValueError(f"images must be [B][3][H][W], got {tuple(x.shape)}")
        with torch.cuda.device(self.device):
            return torch.cat([self._chunk_features(x[i:i + self.max_rows])
                              for i in range(0, x.shape[0], self.max_rows)])

    @torch.no_grad()
    def features_u8(self, x):
        """pool features fp32 [B][2048] on the device of decoded images x u8 [B][H][W][3] (as PIL gives them; pinned
        host memory or the device), pytorch-fid's input path: bit-identical to features(x / 127.5 - 1)"""
        x = torch.as_tensor(x)
        if x.dim() != 4 or x.shape[3] != 3 or x.shape[0] == 0 or x.dtype != torch.uint8:
            raise ValueError(f"images must be uint8 [B][H][W][3], got {x.dtype} {tuple(x.shape)}")
        with torch.cuda.device(self.device):
            return torch.cat([self._chunk_features(x[i:i + self.max_rows], u8=True)
                              for i in range(0, x.shape[0], self.max_rows)])


class FeatureSets:
    """The pool features of a run's sets, collected batch by batch: add(mode, key, image_ids, feats) with key 'origin'
    or a tuple index.  gather() brings every rank's rows to rank 0 sorted by image index (every rank must call it)."""

    def __init__(self):
        self.rows = {}  # (mode, key) -> [(image ids int64 [b], feats fp32 [b][d] on the host)]

    def add(self, mode, key, image_ids, feats):
        self.rows.setdefault((mode, key), []).append(
            (torch.as_tensor(list(image_ids), dtype=torch.int64), feats.detach().float().cpu()))

    def local(self):
        """(mode, key) -> (ids, feats) of this rank's rows, sorted by image index"""
        return {k: _sorted_rows(v) for k, v in self.rows.items()}

    def gather(self, rank=0, world=1):
        """rank 0: (mode, key) -> (ids, feats) of all ranks' rows sorted by image index; other ranks: None"""
        if world == 1:
            return self.local()
        import torch.distributed as dist
        got = [None] * world if rank == 0 else None
        dist.gather_object(self.rows, got, dst=0)
        if rank != 0:
            return None
        merged = {}
        for part in got:
            for k, v in part.items():
                merged.setdefault(k, []).extend(v)
        return {k: _sorted_rows(v) for k, v in merged.items()}


def _sorted_rows(parts):
    ids = torch.cat([p[0] for p in parts])
    feats = torch.cat([p[1] for p in parts])
    order = torch.argsort(ids, stable=True)
    if len(set(ids.tolist())) != ids.numel():
        raise ValueError(f"FID: an image index occurs twice in one set: {sorted(ids.tolist())}")
    return ids[order], feats[order]


# ---- python -m asyrp_official_b200.fid --save-stats DIR OUT.npz: the statistics of a folder of real images ----
IMAGE_EXTENSIONS = ("bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp")  # pytorch-fid's


def image_files(folder):
    """the image files directly in folder with one of pytorch-fid's extensions (as its glob: lower case), sorted"""
    return sorted(os.path.join(folder, f) for f in os.listdir(folder)
                  if f.rsplit(".", 1)[-1] in IMAGE_EXTENSIONS and "." in f and os.path.isfile(os.path.join(folder, f)))


class ImageFiles(torch.utils.data.Dataset):
    """(index, u8 [H][W][3]) of each file, decoded as pytorch-fid decodes it: Image.open(p).convert('RGB') at its own
    size"""

    def __init__(self, files):
        self.files = files

    def __len__(self):
        return len(self.files)

    def __getitem__(self, i):
        from PIL import Image
        with Image.open(self.files[i]) as im:
            return i, torch.from_numpy(np.array(im.convert("RGB"), dtype=np.uint8))


def collate_by_size(items):
    """a loader batch as [(indices int64 [b], u8 [b][H][W][3])], one entry per image size in order of first occurrence"""
    groups = {}
    for i, a in items:
        groups.setdefault(tuple(a.shape), []).append((i, a))
    return [(torch.tensor([i for i, _ in g]), torch.stack([a for _, a in g])) for g in groups.values()]


def folder_features(net, files, batch_size=50, num_workers=8):
    """(pool features fp32 [N][2048] on the device in file order, seconds waiting on the decoding workers, seconds of
    GPU work): each loader batch decoded in DataLoader workers into pinned u8, grouped by size, through features_u8.
    An image's features do not depend on its batch, so neither do the result's bits."""
    loader = torch.utils.data.DataLoader(ImageFiles(files), batch_size=batch_size, num_workers=num_workers,
                                         collate_fn=collate_by_size, pin_memory=True)
    feats = torch.empty(len(files), DIMS, dtype=torch.float32, device=net.device)
    wait = gpu = 0.0
    t0 = time.perf_counter()
    for groups in loader:
        t1 = time.perf_counter()
        for ids, u8 in groups:
            feats[ids.to(net.device)] = net.features_u8(u8)
        torch.cuda.synchronize(net.device)
        t2 = time.perf_counter()
        wait, gpu, t0 = wait + t1 - t0, gpu + t2 - t1, t2
    return feats, wait, gpu


def main(argv=None):
    """--save-stats DIR OUT.npz: the reference statistics (mu, sigma, features, kid_kxx) of the images in DIR; prints
    N and where the time went.  Raises ValueError before any model load on a bad argument."""
    ap = argparse.ArgumentParser(prog="python -m asyrp_official_b200.fid",
                                 description="FID / KID reference statistics of a folder of real images (pytorch-fid's "
                                             "--save-stats, on this library's kernels)")
    ap.add_argument("--save-stats", nargs=2, metavar=("DIR", "OUT"), required=True,
                    help="images directly in DIR (pytorch-fid's extensions, each at its own size) -> OUT (.npz)")
    ap.add_argument("--fid_weights", required=True, help="pytorch-fid's pt_inception-2015-12-05-6726825d.pth")
    ap.add_argument("--batch_size", type=int, default=50)
    ap.add_argument("--num_workers", type=int, default=8)
    a = ap.parse_args(argv)
    folder, out = a.save_stats
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("--save-stats runs single-process: do not launch it under torchrun (WORLD_SIZE > 1)")
    if a.batch_size < 1 or a.num_workers < 0:
        raise ValueError(f"--batch_size must be >= 1 and --num_workers >= 0, got {a.batch_size}, {a.num_workers}")
    if not os.path.isdir(folder):
        raise ValueError(f"--save-stats: {folder!r} is not a directory")
    files = image_files(folder)
    if len(files) < 2:
        raise ValueError(f"--save-stats: {folder!r} holds {len(files)} image file(s) with the extensions "
                         f"{IMAGE_EXTENSIONS}; the statistics need at least 2")
    if not os.path.isfile(a.fid_weights):
        raise ValueError(f"--fid_weights {a.fid_weights!r} is not a file")
    net = FIDInception(a.fid_weights)
    feats, wait, gpu = folder_features(net, files, a.batch_size, a.num_workers)
    t0 = time.perf_counter()
    save_stats(out, feats)
    stats = time.perf_counter() - t0
    print(f"--save-stats: {len(files)} images of {folder} -> {out}; waiting on decoding {wait:.2f} s, features on the "
          f"GPU {gpu:.2f} s, statistics and file {stats:.2f} s")
    return 0


if __name__ == "__main__":
    sys.exit(main())
