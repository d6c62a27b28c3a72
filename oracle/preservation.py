"""fp64 numpy restatement of the content-preservation scores (asyrp_official_b200/preservation.py): save_image's u8
quantisation, PSNR, SSIM and MS-SSIM.  LPIPS is oracle/lpips.py's.  Test infrastructure only; the product never
imports it."""
import numpy as np

WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
WIN, SIGMA = 11, 1.5
C1, C2 = 0.01 ** 2, 0.03 ** 2


def quantize(x):
    """u8 [..] of fp32 x: (x + 1) * 0.5 * 255 + 0.5 with every operation rounded to fp32, clamped to [0, 255],
    truncated (torchvision's save_image after Asyrp.save_image's (x + 1) * 0.5)"""
    x = np.asarray(x, dtype=np.float32)
    t = ((x + np.float32(1)) * np.float32(0.5)) * np.float32(255) + np.float32(0.5)
    return np.trunc(np.clip(t, np.float32(0), np.float32(255))).astype(np.uint8)


def window():
    """the 11 normalised taps exp(-k^2 / (2 sigma^2)), k = -5 .. 5"""
    k = np.arange(WIN, dtype=np.float64) - WIN // 2
    g = np.exp(-(k * k) / (2.0 * SIGMA * SIGMA))
    return g / g.sum()


def filter_valid(x):
    """the window along the last two axes of x without padding: [..][H - 10][W - 10]"""
    g = window()
    H, W = x.shape[-2:]
    h = sum(g[k] * x[..., :, k:k + W - WIN + 1] for k in range(WIN))
    return sum(g[k] * h[..., k:k + H - WIN + 1, :] for k in range(WIN))


def ssim_maps(x, y):
    """(ssim map, cs map) of fp64 planes x, y [..][H][W]"""
    mx, my = filter_valid(x), filter_valid(y)
    sxx = filter_valid(x * x) - mx * mx
    syy = filter_valid(y * y) - my * my
    sxy = filter_valid(x * y) - mx * my
    cs = (2 * sxy + C2) / (sxx + syy + C2)
    return (2 * mx * my + C1) / (mx * mx + my * my + C1) * cs, cs


def ssim_stats(x, y):
    """[..][2]: (mean ssim, mean cs) over the valid pixels of each plane"""
    s, cs = ssim_maps(x, y)
    return np.stack([s.mean((-2, -1)), cs.mean((-2, -1))], -1)


def pool2(x):
    """avg_pool2d(x, 2, stride 2, padding (H mod 2, W mod 2)) over the last two axes, padding counted in the divisor"""
    H, W = x.shape[-2:]
    ph, pw = H % 2, W % 2
    p = np.zeros(x.shape[:-2] + (H + 2 * ph, W + 2 * pw))
    p[..., ph:ph + H, pw:pw + W] = x
    Ho, Wo = (H + 2 * ph - 2) // 2 + 1, (W + 2 * pw - 2) // 2 + 1
    p = p[..., :2 * Ho, :2 * Wo]
    return (p[..., 0::2, 0::2] + p[..., 0::2, 1::2] + p[..., 1::2, 0::2] + p[..., 1::2, 1::2]) / 4


def level_stats(x, y):
    """[5][..][2]: ssim_stats of the five MS-SSIM levels of planes x, y"""
    out = []
    for lvl in range(len(WEIGHTS)):
        out.append(ssim_stats(x, y))
        if lvl < len(WEIGHTS) - 1:
            x, y = pool2(x), pool2(y)
    return np.stack(out)


def psnr(q_src, q_edit):
    """10 log10(255^2 * N / SSE) over the N u8 values of each row ([n][..]); inf where they are equal"""
    d = q_src.astype(np.int64) - q_edit.astype(np.int64)
    sse = (d * d).reshape(d.shape[0], -1).sum(1)
    with np.errstate(divide="ignore"):
        return 10.0 * np.log10(255.0 ** 2 * d[0].size / sse.astype(np.float64))


def scores(src, edited):
    """fp64 [n][3]: (PSNR, SSIM, MS-SSIM) of edited row j (fp32 [n][3][H][W] in [-1, 1]) against src row j % B"""
    qs, qe = quantize(src), quantize(edited)
    qs = qs[np.arange(qe.shape[0]) % qs.shape[0]]
    st = level_stats(qs / 255.0, qe / 255.0)  # [5][n][3][2]
    ms = np.ones(st.shape[1:3])
    for lvl, w in enumerate(WEIGHTS):
        ms = ms * np.maximum(st[lvl, ..., 1] if lvl < len(WEIGHTS) - 1 else st[lvl, ..., 0], 0.0) ** w
    return np.stack([psnr(qs, qe), st[0, ..., 0].mean(-1), ms.mean(-1)], -1)
