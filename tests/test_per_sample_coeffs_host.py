"""Host-side pieces of per-sample DeltaBlock coefficients: the C-ABI layout of AsyrpConvDesc.scales_stride against the
header, the hs_coeff table -> epilogue pair mapping and its validation, and save_image's sweep plan (chunks of whole
hs_coeff tuples, padding rows, the order of the noise draws).  No GPU needed."""
import ctypes
import os
import subprocess

import pytest
import torch

from asyrp_official_b200 import _lib, engine
from asyrp_official_b200.diffusion_latent import chunk_noise, pad_rows, plan_sweep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "asyrp_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu\n", sizeof(AsyrpConvDesc), offsetof(AsyrpConvDesc, scales),
         offsetof(AsyrpConvDesc, sums_out), offsetof(AsyrpConvDesc, scales_stride));
  return 0;
}
"""


def test_conv_desc_layout_matches_the_header(tmp_path):
    """the ctypes mirror of AsyrpConvDesc has the size and field offsets a C compiler gives the header's struct, with
    scales_stride as its last field"""
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(_PROBE)
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, off_scales, off_sums, off_stride = map(int, subprocess.run([str(exe)], capture_output=True, text=True,
                                                                     check=True).stdout.split())
    D = _lib.AsyrpConvDesc
    assert ctypes.sizeof(D) == size
    assert (D.scales.offset, D.sums_out.offset, D.scales_stride.offset) == (off_scales, off_sums, off_stride)
    assert D._fields_[-1][0] == "scales_stride"
    assert D().scales_stride == 0  # a zero-initialised descriptor keeps the shared-pair meaning


def test_coefficient_rows_to_epilogue_pairs():
    """row n = (c0, c1, .., c_k): DeltaBlock i of sample n scales its conv by c_{i+1} and its residual by c0 (i = 0) or
    1 (i > 0); a tuple broadcast to every row gives the pairs set_coeffs has always written"""
    t = torch.tensor([[1.0, 0.5, -2.0], [0.25, 1.5, 3.0]])
    p = engine.coef_pairs(t, 2)
    assert p.shape == (2, 2, 2)
    assert p.tolist() == [[[0.5, 1.0], [-2.0, 1.0]], [[1.5, 0.25], [3.0, 1.0]]]
    one = engine.coef_pairs(torch.tensor([[0.9, 1.3]]), 1)
    assert torch.equal(one, torch.tensor([[[1.3, 0.9]]]))


def test_coefficient_table_validation():
    assert engine.coeff_table([[1.0, 0.5], [1.0, 2.0]], 2, 1).dtype == torch.float32
    for bad in ([[1.0, 0.5]], [[1.0, 0.5, 0.1], [1.0, 2.0, 0.2]], [1.0, 0.5], torch.ones(2, 2, dtype=torch.int32)):
        with pytest.raises(_lib.AsyrpError):
            engine.coeff_table(bad, 2, 1)
    assert engine.shared_c0(torch.tensor([[0.6, 1.0], [0.6, 2.0]])) == float(torch.tensor(0.6))
    with pytest.raises(_lib.AsyrpError):
        engine.shared_c0(torch.tensor([[0.6, 1.0], [1.0, 2.0]]))


@pytest.mark.parametrize("n_tuples,bs,max_rows,tpc,chunks", [
    (5, 1, 16, 5, [[0, 1, 2, 3, 4]]),              # one chunk, no padding beyond the tuples
    (5, 1, 1, 1, [[0], [1], [2], [3], [4]]),      # one replay per tuple
    (5, 4, 16, 4, [[0, 1, 2, 3], [4]]),            # 16 rows, the last chunk padded from 4 to 16 rows
    (3, 2, 4, 2, [[0, 1], [2]]),
    (3, 32, 16, 1, [[0], [1], [2]]),              # a batch larger than the bound still runs whole tuples
    (25, 1, 16, 16, [list(range(16)), list(range(16, 25))]),
])
def test_sweep_chunks(n_tuples, bs, max_rows, tpc, chunks):
    assert plan_sweep(n_tuples, bs, max_rows) == (tpc, chunks)


def test_padding_rows_repeat_the_last_row():
    x = torch.arange(6.0).reshape(3, 2)
    p = pad_rows(x, 5)
    assert p.tolist() == [[0, 1], [2, 3], [4, 5], [4, 5], [4, 5]]
    assert pad_rows(x, 3) is x


def test_noise_draws_follow_the_per_tuple_order():
    """a chunk's noise is the per-tuple draws of the sequential loop, in tuple order, along the batch axis; padding rows
    copy the last real row and consume nothing from the generator"""
    n_sto, bs, shape = 3, 2, (3, 4, 4)
    seq_gen = torch.Generator().manual_seed(5)
    sequential = [torch.randn((n_sto, bs, *shape), generator=seq_gen) for _ in range(3)]
    after_seq = torch.randn(1, generator=seq_gen)
    gen = torch.Generator().manual_seed(5)
    draw = lambda: torch.randn((n_sto, bs, *shape), generator=gen)  # noqa: E731
    z1 = chunk_noise(2, 2, bs, draw)   # tuples 0, 1
    z2 = chunk_noise(1, 2, bs, draw)   # tuple 2, padded to two tuples' rows
    assert z1.shape == z2.shape == (n_sto, 2 * bs, *shape)
    assert torch.equal(z1, torch.cat(sequential[:2], dim=1))
    assert torch.equal(z2[:, :bs], sequential[2])
    assert torch.equal(z2[:, bs:], sequential[2][:, -1:].expand(n_sto, bs, *shape))
    assert torch.equal(torch.randn(1, generator=gen), after_seq)
