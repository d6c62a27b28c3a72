"""scoring.Scorers.score with stub networks on the CPU: what one batch writes (the score TSVs) and keeps (the runner's
score dicts and the FID feature sets) for a single edit, an hs_coeff interpolation and an attribute sweep, and how
directional CLIP is called in each.  No GPU needed."""
import csv
import os

import pytest
import torch

from asyrp_official_b200 import fid, main as cli
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.scoring import Scorers

BS = 2


class Stub:
    """every scorer method returns seeded values, one per edited row; directional CLIP's calls are recorded"""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)
        self.clip_calls = []

    def _rows(self, edited, *shape, dtype=torch.float32):
        return torch.rand(edited.shape[0], *shape, generator=self.g, dtype=dtype)

    def directional_similarity(self, origin, src, edited, trg):
        self.clip_calls.append((src, trg, edited.shape[0]))
        return self._rows(edited)

    def id_similarity(self, origin, edited):
        return self._rows(edited)

    def seg_consistency(self, origin, edited):
        return self._rows(edited, dtype=torch.float64)

    def scores(self, src, edited):
        return self._rows(edited, 4, dtype=torch.float64)

    def features(self, x):
        return self._rows(x, 8)


def _table(path):
    with open(path) as f:
        return list(csv.reader(f, delimiter="\t"))


def _scorers(tmp_path, monkeypatch, attrs):
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--exp", "./runs/s"])
    s = Scorers(Asyrp(args, cfg, device="cpu"), attrs)  # no score flags: nothing to check or build
    assert not s.needs_origin and not s.nets
    s.nets = {name: Stub(seed) for seed, name in enumerate(("clip", "id", "seg", "fid", "cp"))}
    s.texts = (["face", "face"], ["smiling face", "angry face"]) if attrs else ("face", "smiling face")
    s.fid_sets = fid.FeatureSets()
    os.makedirs("out")  # save_image's folder, made before it scores
    return s


@pytest.mark.parametrize("mode", ["single", "interp", "sweep"])
def test_score_writes_and_keeps_every_score(tmp_path, monkeypatch, mode):
    attrs = ["smiling", "angry"] if mode == "sweep" else None
    coeffs = {"single": [(1.0, 0.5)], "interp": [(1.0, 0.25), (1.0, 0.5), (1.0, 1.5)],
              "sweep": [(1.0, 0.5, 0.0), (1.0, 0.0, 0.5)]}[mode]
    s = _scorers(tmp_path, monkeypatch, attrs)
    r = s.runner
    g = torch.Generator().manual_seed(9)
    origin = torch.rand(BS, 3, 8, 8, generator=g)
    edited = [torch.rand(BS, 3, 8, 8, generator=g) for _ in coeffs]
    source = torch.rand(BS, 3, 8, 8, generator=g)
    s.score("test_1_0", "out", "test", [0, 1], origin, edited, coeffs, source)
    s.score("test_3_0", "out", "test", [2, 3], origin, edited, coeffs)  # latents not inverted from images
    n = len(coeffs)
    # directional CLIP: one call over every tuple with the shared text pair, or one per attribute with its own texts
    want = [("face", "smiling face", n * BS)] if attrs is None else [("face", "smiling face", BS),
                                                                       ("face", "angry face", BS)]
    assert s.nets["clip"].clip_calls == want * 2
    for name, column, shape in (("directional_clip", ["S_dir"], (n, BS)), ("id_similarity", ["ID"], (n, BS)),
                                ("seg_consistency", ["SC"], (n, BS)),
                                ("content_preservation", ["PSNR", "SSIM", "MS_SSIM", "LPIPS"], (n, BS, 4))):
        kept = getattr(r, name)["test_1_0"]
        assert kept.shape == shape
        t = _table(os.path.join("out", f"test_1_0_ngen6_{name}.tsv"))
        assert t[0] == ["image", "tuple", "hs_coeff"] + column + (["attr"] if attrs else [])
        rows = t[1:]
        if name == "content_preservation":  # the origin pass against the input images comes first
            rec = r.reconstruction["test_1_0"]
            assert [row[:3] for row in rows[:BS]] == [[str(i), "origin", "-"] for i in range(BS)]
            assert torch.equal(torch.tensor([[float(v) for v in row[3:7]] for row in rows[:BS]], dtype=torch.float64),
                               rec)
            rows = rows[BS:]
        assert [row[:3] for row in rows] == [[str(i), str(k), ",".join(f"{c:.6g}" for c in coeffs[k])]
                                             for k in range(n) for i in range(BS)]
        if attrs:
            assert [row[-1] for row in t[1:]] == ["-"] * (BS if name == "content_preservation" else 0) + \
                [a for a in attrs for _ in range(BS)]
        vals = torch.tensor([[float(v) for v in row[3:3 + len(column)]] for row in rows], dtype=torch.float64)
        assert torch.equal(vals.view(shape), kept.double())
    assert "test_3_0" not in r.reconstruction and "test_3_0" in r.content_preservation
    assert _table(os.path.join("out", "test_3_0_ngen6_content_preservation.tsv"))[1][1] == "0"
    # --fid: the origin rows and each tuple's rows, with the batch's image indices
    got = s.fid_sets.gather()
    assert set(got) == {("test", "origin")} | {("test", k) for k in range(n)}
    assert all(torch.equal(ids, torch.arange(4)) and f.shape == (4, 8) for ids, f in got.values())


def test_score_without_edits_or_scores_writes_nothing(tmp_path, monkeypatch):
    s = _scorers(tmp_path, monkeypatch, None)
    s.score("test_1_0", "out", "test", [0, 1], torch.zeros(BS, 3, 8, 8), [], [(1.0, 0.5)], torch.zeros(BS, 3, 8, 8))
    assert os.listdir("out") == [] and not s.runner.directional_clip and s.fid_sets.gather() == {}
    s.nets = {}  # a run without score flags: save_image runs no origin pass
    s.score("test_1_0", "out", "test", [0, 1], None, [torch.zeros(BS, 3, 8, 8)], [(1.0, 0.5)])
    assert os.listdir("out") == []
