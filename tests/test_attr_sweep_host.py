"""Host-side pieces of attribute sweeps: RowSchedule's per-row tables against the single-row Schedules, the gating
coefficients below each row's t_edit, the engine's row bookkeeping, the sweep's chunks / grid rows / score columns,
every refusal of --attr_sweep and the flag's parsing.  No GPU needed."""
import csv
import os

import pytest
import torch

from asyrp_official_b200 import _lib, engine, main as cli
from asyrp_official_b200.diffusion_latent import Asyrp, plan_sweep, sweep_rows
from asyrp_official_b200.scoring import write_scores
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences
from oracle import sampler as osmp

T_EDIT, T_ADD = [700, 500, 300, 10 ** 9], [0, 450, 650, 0]
COEFFS = [(1.0, 1.0, 0.0, 0.0), (1.0, 0.0, 1.25, 0.0), (0.9, 0.0, 0.0, -0.7), (1.0, 1.0, 0.0, 0.0)]


def _rs(n_step=8, **kw):
    seq, seq_next = make_sequences(999, n_step)
    return RowSchedule(osmp.make_betas(), seq, seq_next, T_EDIT, T_ADD, COEFFS, **kw), seq, seq_next


def test_row_tables_equal_the_single_row_schedules():
    rs, seq, seq_next = _rs()
    assert rs.c.shape == (len(rs.steps), 4, 2) and rs.coeffs.shape == (len(rs.steps), 4, 4)
    for n in range(4):
        one = Schedule(osmp.make_betas(), seq, seq_next, t_edit=T_EDIT[n], t_addnoise=T_ADD[n], hs_coeff=COEFFS[n])
        for k, (s, o) in enumerate(zip(rs.steps, one.steps)):
            assert (s.t, s.t_next, s.at, s.an) == (o.t, o.t_next, o.at, o.an)
            assert rs.c[k, n, 0].item() == o.c1 and rs.c[k, n, 1].item() == o.c2
            assert s.edit_rows[n] == o.edit
            want = COEFFS[n] if o.edit else (1.0, 0.0, 0.0, 0.0)
            assert tuple(rs.coeffs[k, n].tolist()) == tuple(torch.tensor(want, dtype=torch.float32).tolist())
    for s in rs.steps:
        assert s.edit == any(s.edit_rows)
    singles = [Schedule(osmp.make_betas(), seq, seq_next, t_edit=T_EDIT[n], t_addnoise=T_ADD[n]) for n in range(4)]
    assert [s.stochastic for s in rs.steps] == [any(o.steps[k].stochastic for o in singles)
                                                for k in range(len(rs.steps))]
    assert rs.n_stochastic == sum(s.stochastic for s in rs.steps) > 0
    assert rs.n_edit == sum(s.edit for s in rs.steps)


def test_gating_below_t_edit_and_never_edited_rows():
    rs, _, _ = _rs()
    for k, s in enumerate(rs.steps):
        for n in range(4):
            if s.t < T_EDIT[n]:
                assert rs.coeffs[k, n].tolist() == [1.0, 0.0, 0.0, 0.0] and not s.edit_rows[n]
    assert not any(s.edit_rows[3] for s in rs.steps)  # t_edit above every step


def test_noise_rows_are_the_single_row_draws():
    rs, seq, seq_next = _rs()
    nz = torch.arange(rs.n_stochastic * 4, dtype=torch.float32).view(rs.n_stochastic, 4)
    for n in range(4):
        one = Schedule(osmp.make_betas(), seq, seq_next, t_edit=T_EDIT[n], t_addnoise=T_ADD[n])
        got = rs.noise_rows(n, nz)
        assert tuple(got.shape) == (one.n_stochastic, 1)
        sto = [s.t for s in rs.steps if s.stochastic]
        assert [sto[int(v) // 4] for v in got[:, 0].tolist()] == [s.t for s in one.steps if s.stochastic]
        assert all(int(v) % 4 == n for v in got[:, 0].tolist())


def test_row_schedule_refusals_and_graph_key():
    seq, seq_next = make_sequences(999, 4)
    b = osmp.make_betas()
    with pytest.raises(ValueError):
        RowSchedule(b, seq, seq_next, [500], [0], [(1.0, 1.0)], sample_type="ddpm")
    with pytest.raises(ValueError):
        RowSchedule(b, seq, seq_next, [500, 400], [0], [(1.0, 1.0), (1.0, 1.0)])
    with pytest.raises(ValueError):
        RowSchedule(b, seq, seq_next, [500, 400], [0, 0], [(1.0, 1.0), (1.0, 1.0, 0.0)])
    a = RowSchedule(b, seq, seq_next, [500, 400], [0, 0], [(1.0, 1.0), (1.0, 2.0)])
    same = RowSchedule(b, seq, seq_next, [500, 400], [0, 0], [(1.0, 3.0), (1.0, 0.5)])
    assert a.key() == same.key()  # coefficients are device-side tables
    assert a.key() != RowSchedule(b, seq, seq_next, [500, 100], [0, 0], [(1.0, 1.0), (1.0, 2.0)]).key()


def test_engine_row_bookkeeping():
    pairs = engine.sweep_pairs(torch.tensor([[0.75, 0.0, 1.5], [1.0, 2.0, 0.0]]))
    assert pairs.tolist() == [[[0.0, 0.75], [1.5, 0.75]], [[2.0, 1.0], [0.0, 1.0]]]
    assert engine.sweep_pairs(torch.zeros(3, 2, 4)).shape == (3, 2, 3, 2)
    assert engine.own_blocks(COEFFS) == (0, 1, 2, 0)
    assert engine.own_blocks([(1.0, 0.0, 0.0)]) == (0,)
    with pytest.raises(_lib.AsyrpError):
        engine.own_blocks([(1.0, 0.5, 0.5)])
    assert engine.row_runs([1, 1, 2, 2, 2, 1]) == [(0, 2, 1), (2, 5, 2), (5, 6, 1)]
    assert engine.row_runs([(True, 0)]) == [(0, 1, (True, 0))]


def test_chunks_and_grid_rows():
    # 3 attributes x 2 images: rows attribute-major; 4 rows per replay -> chunks of 2 attributes, the last padded
    tpc, chunks = plan_sweep(3, 2, 4)
    assert (tpc, chunks) == (2, [[0, 1], [2]])
    assert sweep_rows(chunks[0], tpc, 2) == [0, 0, 1, 1]
    assert sweep_rows(chunks[1], tpc, 2) == [2, 2, 2, 2]
    assert plan_sweep(8, 1, 16) == (8, [list(range(8))])
    assert sweep_rows(list(range(3)), 3, 1) == [0, 1, 2]


def test_score_table_names_the_attribute(tmp_path):
    coeffs = [(1.0, 0.5, 0.0), (1.0, 0.0, 0.5)]
    p = str(tmp_path / "s.tsv")
    write_scores(p, coeffs, torch.tensor([[0.1, 0.2], [0.3, 0.4]]), "ID", "identity similarity",
                 attrs=["smiling", "angry"])
    with open(p) as f:
        t = list(csv.reader(f, delimiter="\t"))
    assert t[0] == ["image", "tuple", "hs_coeff", "ID", "attr"]
    assert [(r[0], r[1], r[2], r[4]) for r in t[1:]] == [("0", "0", "1,0.5,0", "smiling"), ("1", "0", "1,0.5,0", "smiling"),
                                                         ("0", "1", "1,0,0.5", "angry"), ("1", "1", "1,0,0.5", "angry")]
    write_scores(p, coeffs, torch.tensor([[0.1], [0.3]]), "ID", "identity similarity")
    with open(p) as f:
        assert next(csv.reader(f, delimiter="\t")) == ["image", "tuple", "hs_coeff", "ID"]


# ------------------------------------------------------------------------------------------------------------------
# CLI
# ------------------------------------------------------------------------------------------------------------------
def _runner(tmp_path, monkeypatch, extra):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint", exist_ok=True)
    for a in ("smiling", "angry"):
        torch.save({"0": {}}, f"checkpoint/{a}_0.pth")
    argv = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/s", "--train_delta_block", "--get_h_num", "1",
            "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "200", "--attr_sweep", "smiling angry",
            "--manual_checkpoint_name", "attribute_0.pth"] + extra
    args, config = cli.parse_args_and_config(argv)
    return Asyrp(args, config, device="cpu")


def test_attr_sweep_setup_resolves_one_checkpoint_per_attribute(tmp_path, monkeypatch):
    r = _runner(tmp_path, monkeypatch, [])
    attrs, paths = r.attr_sweep_setup()
    assert attrs == ["smiling", "angry"]
    assert paths == [os.path.join("checkpoint", "smiling_0.pth"), os.path.join("checkpoint", "angry_0.pth")]
    assert r.attr_sweep_schedules(attrs) == [(500, 200), (500, 200)]


@pytest.mark.parametrize("extra", [
    ["--multiple_attr", "smiling angry"], ["--delta_interpolation"], ["--num_mean_of_delta_hs", "2"],
    ["--train_delta_h"], ["--sample_type", "ddpm"], ["--get_h_num", "2"], ["--get_h_num", "0"],
    ["--attr_sweep", "smiling sad"], ["--manual_checkpoint_name", "smiling_0.pth"], ["--attr_sweep", "smiling smiling"]])
def test_attr_sweep_refusals_before_any_model_loads(tmp_path, monkeypatch, extra):
    r = _runner(tmp_path, monkeypatch, extra)

    def no_model():
        raise AssertionError("a model was loaded")

    monkeypatch.setattr(r, "load_pretrained_model", no_model)
    with pytest.raises(ValueError):
        r.run_test()


def test_flags_parse(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    args, _ = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--attr_sweep", "smiling angry young"])
    assert args.attr_sweep == "smiling angry young"
    plain, _ = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--edit_attr", "smiling",
                                          "--multiple_attr", "a b", "--max_rows_per_replay", "4"])
    assert plain.attr_sweep == "" and plain.edit_attr == "smiling" and plain.multiple_attr == "a b"
    assert plain.max_rows_per_replay == 4 and plain.get_h_num == 0
