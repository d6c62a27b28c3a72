"""CPU oracle of the FID Inception-v3 pool features and of FID / KID (asyrp_official_b200/fid.py gives the network and
the metric, this project's definition).  Test infrastructure only; evaluated in fp64 by default (the `dtype` argument).

The blocks the FID variant shares with torchvision's Inception3 (the stem, InceptionB as Mixed_6a, InceptionD as
Mixed_7a) are torchvision's own modules; the four FID blocks are written out from pytorch-fid's public definition:
FIDInceptionA / C / E_1 pool with avg_pool2d(3, 1, 1, count_include_pad=False), FIDInceptionE_2 with max_pool2d(3, 1, 1).
frechet_distance_sqrtm restates pytorch-fid's calculate_frechet_distance (scipy.linalg.sqrtm of S1 S2).
"""
import types

import numpy as np
import torch
import torch.nn.functional as F

SIZE = 299


def quantise(x):
    """the u8 values torchvision's save_image writes for an image x in [-1, 1] (fp32: (x + 1) * 0.5, * 255, + 0.5,
    clamped, truncated), as uint8"""
    t = (x.float() + 1) * 0.5
    return t.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)


def preprocess(x, dtype=torch.float64):
    """pytorch-fid's input for the PNG of x: u8 / 255 (ToTensor), bilinear 299 x 299 (align_corners=False), 2 v - 1"""
    v = quantise(x).to(torch.float32) / 255
    v = F.interpolate(v, size=(SIZE, SIZE), mode="bilinear", align_corners=False)
    return (2 * v - 1).to(dtype)


def _fid_a(self, x):
    b1 = self.branch1x1(x)
    b5 = self.branch5x5_2(self.branch5x5_1(x))
    b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
    bp = self.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
    return torch.cat([b1, b5, b3, bp], 1)


def _fid_c(self, x):
    b1 = self.branch1x1(x)
    b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
    bd = self.branch7x7dbl_1(x)
    for k in range(2, 6):
        bd = getattr(self, f"branch7x7dbl_{k}")(bd)
    bp = self.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
    return torch.cat([b1, b7, bd, bp], 1)


def _fid_e(pool):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b3 = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(b3), self.branch3x3_2b(b3)], 1)
        bd = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = torch.cat([self.branch3x3dbl_3a(bd), self.branch3x3dbl_3b(bd)], 1)
        bp = self.branch_pool(pool(x))
        return torch.cat([b1, b3, bd, bp], 1)
    return forward


FID_FORWARD = {
    "A": _fid_a, "C": _fid_c,
    "E1": _fid_e(lambda x: F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)),
    "E2": _fid_e(lambda x: F.max_pool2d(x, kernel_size=3, stride=1, padding=1)),
}
FID_BLOCKS = {"Mixed_5b": "A", "Mixed_5c": "A", "Mixed_5d": "A", "Mixed_6b": "C", "Mixed_6c": "C", "Mixed_6d": "C",
              "Mixed_6e": "C", "Mixed_7b": "E1", "Mixed_7c": "E2"}


def torchvision_inception(sd, dtype=torch.float64):
    """torchvision's Inception3 (aux_logits False, 1008 classes) in eval mode holding the state dict sd, unmodified"""
    from torchvision.models.inception import Inception3
    m = Inception3(num_classes=1008, aux_logits=False, transform_input=False, init_weights=False)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    if unexpected or any(not (k.startswith("fc.") or k.endswith("num_batches_tracked")) for k in missing):
        raise ValueError(f"oracle: state dict does not match Inception3: missing {missing}, unexpected {unexpected}")
    return m.to(dtype).eval()


def fid_inception(sd, dtype=torch.float64):
    """torchvision_inception with the FID blocks' forward"""
    m = torchvision_inception(sd, dtype)
    for name, kind in FID_BLOCKS.items():
        blk = getattr(m, name)
        blk.forward = types.MethodType(FID_FORWARD[kind], blk)
    return m


def stem(m, x):
    """Conv2d_1a .. Conv2d_4a and both max-pools: [B][192][35][35] from the 299^2 input"""
    x = m.Conv2d_2b_3x3(m.Conv2d_2a_3x3(m.Conv2d_1a_3x3(x)))
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    x = m.Conv2d_4a_3x3(m.Conv2d_3b_1x1(x))
    return F.max_pool2d(x, kernel_size=3, stride=2)


@torch.no_grad()
def features(m, x):
    """pool features [B][2048] of the preprocessed input x [B][3][299][299]"""
    x = stem(m, x)
    for name in ("Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e",
                 "Mixed_7a", "Mixed_7b", "Mixed_7c"):
        x = getattr(m, name)(x)
    return x.mean(dim=(2, 3))


def frechet_distance_sqrtm(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """pytorch-fid's calculate_frechet_distance: |mu1 - mu2|^2 + tr S1 + tr S2 - 2 tr sqrtm(S1 S2), with its offset
    retry on a singular product and its check that the imaginary part is negligible"""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))  # pytorch-fid passes disp=False, which newer scipy no longer takes
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def moments(f):
    """mu and np.cov (n - 1 denominator) of features [n][d], fp64"""
    f = np.asarray(f, dtype=np.float64)
    return f.mean(axis=0), np.cov(f, rowvar=False)


def kid_loop(f1, f2):
    """the unbiased MMD^2 with k(x, y) = (x . y / d + 1)^3 as a direct double loop over the rows (fp64)"""
    f1, f2 = np.asarray(f1, dtype=np.float64), np.asarray(f2, dtype=np.float64)
    n, m, d = f1.shape[0], f2.shape[0], f1.shape[1]

    def k(a, b):
        return (a @ b / d + 1) ** 3

    sxx = sum(k(f1[i], f1[j]) for i in range(n) for j in range(n) if i != j)
    syy = sum(k(f2[i], f2[j]) for i in range(m) for j in range(m) if i != j)
    sxy = sum(k(f1[i], f2[j]) for i in range(n) for j in range(m))
    return sxx / (n * (n - 1)) + syy / (m * (m - 1)) - 2 * sxy / (n * m)
