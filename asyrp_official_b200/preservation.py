"""Content preservation of edits: PSNR, SSIM, MS-SSIM and LPIPS of each edited image against its source image, all on
the u8 image torchvision's save_image writes, so that the numbers equal what a user measures from the written PNGs.

    q        the u8 save_image writes for an fp32 image in [-1, 1]: fp32 (x + 1) * 0.5 * 255 + 0.5, clamped to [0, 255],
             truncated (ops.png_quantize, the quantiser of fid.FIDInception)
    PSNR     10 log10(255^2 * 3 H W / SSE), SSE = sum over the three channels of (q_edit - q_src)^2, an exact 64-bit
             integer on the GPU; the log in fp64 on the host; SSE = 0 gives inf
    SSIM     pytorch_msssim.ssim(data_range=1, size_average=False) restated in fp64: x = q / 255 per channel, an 11-tap
             Gaussian window (sigma 1.5, normalised) applied separably without padding, C1 = 0.01^2, C2 = 0.03^2,
             mu = G * x, sigma_x^2 = G * x^2 - mu_x^2, sigma_xy = G * (x y) - mu_x mu_y,
             cs = (2 sigma_xy + C2) / (sigma_x^2 + sigma_y^2 + C2), ssim = (2 mu_x mu_y + C1) / (mu_x^2 + mu_y^2 + C1) cs,
             each map averaged over its valid pixels per channel, then the mean of the three channels.  The same
             quantity as scikit-image's structural_similarity(gaussian_weights=True, sigma=1.5,
             use_sample_covariance=False, data_range=1)
    MS-SSIM  pytorch_msssim.ms_ssim: five levels with WEIGHTS, avg_pool2d(2, stride 2, padding (H mod 2, W mod 2))
             between them (padding counted in the divisor); per channel prod_{l<4} relu(mean cs_l)^w_l *
             relu(mean ssim_4)^w_4, then the mean over the channels.  Needs min(H, W) > (11 - 1) * 2^4 = 160
    LPIPS    the library's LPIPS-Alex (lpips.LPIPS) on (2 q - 255) / 255 in fp32: what the lpips package's im2tensor
             gives for a loaded PNG (q / 127.5 - 1 in fp64, then fp32), up to the last fp32 bit

Edited row j is compared with source row j % B.  Every operation but the per-row combination of the statistics (a few
fp64 operations on the host) is a kernel of libasyrp_b200.so; the SSIM statistics are fp64, so identical images give
exactly PSNR = inf, SSIM = MS-SSIM = 1 and LPIPS = 0, and a row's four scores are the same bits in any batch or chunk.
"""
import numpy as np
import torch

from . import _lib, lpips, ops

COLUMNS = ("PSNR", "SSIM", "MS_SSIM", "LPIPS")
WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
LEVELS = len(WEIGHTS)
WIN = 11
MIN_SIZE = (WIN - 1) * 2 ** (LEVELS - 1) + 1  # 161
# device memory of the scored rows: rows are scored in chunks of at most ACTIVATION_BUDGET // row_bytes(H, W) images
ACTIVATION_BUDGET = 1 << 30


def check_image_size(H, W):
    if min(H, W) < MIN_SIZE:
        raise ValueError(f"MS-SSIM's five levels need images larger than {MIN_SIZE - 1} x {MIN_SIZE - 1}, got {H}x{W}")


def level_shapes(H, W):
    """(H_l, W_l) of the five MS-SSIM levels"""
    out = [(H, W)]
    for _ in range(LEVELS - 1):
        h, w = out[-1]
        out.append(((h + 1) // 2, (w + 1) // 2))
    return out


def row_bytes(H, W):
    """device bytes one scored image holds: its fp32 copy, q, the fp64 pyramid, the LPIPS input and features"""
    pyramid = sum(h * w for h, w in level_shapes(H, W))
    shp = lpips.feature_shapes(H, W)
    feats = H * W * 4 + sum(h * w * c for (h, w), c in zip(shp, lpips.CHANNELS)) + \
        sum(((h - 3) // 2 + 1) * ((w - 3) // 2 + 1) * c for (h, w), c in zip(shp[:2], lpips.CHANNELS[:2]))
    return 3 * H * W * (4 + 1 + 4) + 3 * 8 * pyramid + 4 * feats


def combine(sse, stats, lp, H, W):
    """the four scores, fp64 [n][4], from SSE int64 [n], the level statistics fp64 [LEVELS][n][3][2] (mean ssim, mean
    cs) and LPIPS [n] (numpy arrays)"""
    sse = np.asarray(sse, dtype=np.int64)
    n = sse.shape[0]
    out = np.empty((n, 4), dtype=np.float64)
    with np.errstate(divide="ignore"):
        out[:, 0] = 10.0 * np.log10(255.0 ** 2 * (3 * H * W) / sse.astype(np.float64))
    out[:, 1] = stats[0, :, :, 0].mean(-1)
    ms = np.ones((n, 3), dtype=np.float64)
    for lvl in range(LEVELS):
        v = stats[lvl, :, :, 1] if lvl < LEVELS - 1 else stats[lvl, :, :, 0]
        ms = ms * np.maximum(v, 0.0) ** WEIGHTS[lvl]
    out[:, 2] = ms.mean(-1)
    out[:, 3] = np.asarray(lp, dtype=np.float64)
    return out


class _Rows:
    """device buffers of `rows` images of H x W: the fp32 copy, q, the fp64 pyramid and the LPIPS input"""

    def __init__(self, rows, H, W, device):
        self.x = torch.empty(rows, 3, H, W, dtype=torch.float32, device=device)
        self.q = torch.empty(rows, 3, H, W, dtype=torch.uint8, device=device)
        self.levels = [torch.empty(rows, 3, h, w, dtype=torch.float64, device=device) for h, w in level_shapes(H, W)]
        self.xq = torch.empty(rows, 3, H, W, dtype=torch.float32, device=device)


class ContentPreservation:
    """ContentPreservation(lpips_state_dict_or_path, device, max_rows=None).scores(src, edited): fp64 [n][4] on the
    host, (PSNR, SSIM, MS_SSIM, LPIPS) of edited row j against source row j % B (module docstring).  Owns one
    lpips.LPIPS; device buffers are pooled per shape.  The sources are prepared once; the edited rows run in chunks of
    a whole multiple of B rows, at most max_rows (default ACTIVATION_BUDGET // row_bytes(H, W)) when that is at least
    B, which bounds the memory for any number of edited rows."""

    def __init__(self, lpips_state_dict_or_path, device=None, max_rows=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("ContentPreservation needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        self.lpips = lpips.LPIPS(lpips_state_dict_or_path, device=device)
        self.device = self.lpips.device
        self.max_rows = None if max_rows is None else max(1, int(max_rows))
        self._rows = {}

    def _prepare(self, x, slot):
        """copy x to the pooled buffers of (rows, H, W, slot), quantise, build the pyramid and the LPIPS features"""
        key = (x.shape[0], x.shape[2], x.shape[3], slot)
        if key not in self._rows:
            self._rows[key] = _Rows(*key[:3], self.device)
        b = self._rows[key]
        b.x.copy_(x)
        ops.png_quantize(b.x, b.q, b.levels[0], b.xq)
        for lo, hi in zip(b.levels[:-1], b.levels[1:]):
            ops.ssim_pool2(lo, hi)
        return b, self.lpips.features(b.xq, slot)

    @torch.no_grad()
    def scores(self, src, edited):
        src, edited = torch.as_tensor(src), torch.as_tensor(edited)
        if src.dim() != 4 or src.shape[1] != 3 or edited.dim() != 4 or edited.shape[1:] != src.shape[1:]:
            raise ValueError(f"images must be [B][3][H][W] and [n][3][H][W] of one size, got {tuple(src.shape)} and "
                             f"{tuple(edited.shape)}")
        B, N = src.shape[0], edited.shape[0]
        if B == 0 or N % B:
            raise ValueError(f"edited images ({N}) must be a whole multiple of the source images ({B})")
        H, W = src.shape[2], src.shape[3]
        check_image_size(H, W)
        max_rows = self.max_rows if self.max_rows is not None else ACTIVATION_BUDGET // row_bytes(H, W)
        rows = B * max(1, max_rows // B)  # chunks start at multiples of B: row j pairs with source j % B
        dev = self.device
        with torch.cuda.device(dev):
            s, ref = self._prepare(src, "ref")
            sse = torch.empty(N, dtype=torch.int64, device=dev)
            stats = torch.empty(LEVELS, N, 3, 2, dtype=torch.float64, device=dev)
            lp = torch.empty(N, dtype=torch.float32, device=dev)
            for i in range(0, N, rows):
                c = min(rows, N - i)
                e, probe = self._prepare(edited[i:i + c], "probe")
                ops.preserve_sse(s.q, e.q, sse[i:i + c])
                for lvl in range(LEVELS):
                    ops.ssim_level(s.levels[lvl], e.levels[lvl], stats[lvl, i:i + c])
                self.lpips.distance(probe, ref, lp[i:i + c])
            out = combine(sse.cpu().numpy(), stats.cpu().numpy(), lp.cpu().numpy(), H, W)
        return torch.from_numpy(out)
