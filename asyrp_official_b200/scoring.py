"""The edit scores of `--run_test` (with or without `--attr_sweep`): their requirement checks, the scoring networks of
one run, and the score tables they write.

  per edit  --DirectionalClipSmilarity  clip_image.CLIPLoss           <file>_ngen<n>_directional_clip.tsv
            --id_similarity             arcface.ArcFace               <file>_ngen<n>_id_similarity.tsv
            --seg_consistency           face_parsing.FaceParser       <file>_ngen<n>_seg_consistency.tsv
            --content_preservation      preservation.ContentPreservation  <file>_ngen<n>_content_preservation.tsv
            --dino_structure            dino.DINO                     <file>_ngen<n>_dino.tsv
  per set   --fid (--fid_ref, --prdc)   fid.FIDInception, FeatureSets <mode>_ngen<n>_{fid,fid_real,prdc,prdc_real}.tsv

Every per-edit score compares each edit against the origin pass (the unedited DDIM pass of the same x_T), which
save_image runs once for all of them; --fid collects the pool features of the origin pass and of the edits and scores
the sets at the end of the run.  The checks run before any model loads and raise ValueError with the reason.
"""
import math
import os

import torch


def fid_options_check(runner):
    """--fid_ref's and --prdc's requirements, checked before any other flag of --run_test"""
    a = runner.args
    if getattr(a, "fid_ref", None) is not None and not getattr(a, "fid", False):
        raise ValueError("--fid_ref scores the sets that --fid collects: add --fid")
    runner.prdc_check()


def prdc_check(runner):
    """--prdc's requirements, checked before any model is loaded; raises ValueError with the reason"""
    a = runner.args
    if not getattr(a, "prdc", False):
        return
    if not getattr(a, "fid", False):
        raise ValueError("--prdc scores the pool features that --fid collects: add --fid")
    if not 1 <= a.prdc_k <= 32:
        raise ValueError(f"--prdc: --prdc_k must be in 1..32, got {a.prdc_k}")


def directional_clip_setup(runner, attrs=None):
    """--DirectionalClipSmilarity's requirements; raises ValueError with the reason.  Returns (src_txt, trg_txt,
    templates): src_txts[0] / trg_txts[0] of runner.edit_texts(), the pair run_training scores
    (diffusion_latent.py:343), and imagenet_templates from --text_templates.  With attrs (an attribute sweep) src_txt
    and trg_txt are lists, the pair of each attribute."""
    from .clip_image import read_templates
    a = runner.args
    if getattr(a, "multiple_attr", ""):
        raise ValueError("--DirectionalClipSmilarity scores one source / target text pair: a --multiple_attr edit "
                         "has none")
    if getattr(a, "pass_editing", False):
        raise ValueError("--DirectionalClipSmilarity scores the edited images: with --pass_editing nothing is "
                         "edited")
    if not runner.clip_configured():
        raise ValueError("--DirectionalClipSmilarity needs --clip_weights and --clip_vocab")
    for flag, path in (("--clip_weights", a.clip_weights), ("--clip_vocab", a.clip_vocab)):
        if not os.path.isfile(path):
            raise ValueError(f"--DirectionalClipSmilarity: {flag} {path!r} is not a file")
    try:
        templates = read_templates(getattr(a, "text_templates", None) or os.path.join("utils", "text_templates.py"))
    except FileNotFoundError as e:
        raise ValueError(f"--DirectionalClipSmilarity: {e}") from None
    if attrs is not None:
        texts = [runner.edit_texts(attr) for attr in attrs]
        return [src[0] for src, _ in texts], [trg[0] for _, trg in texts], templates
    src, trg = runner.edit_texts()
    return src[0], trg[0], templates


def id_similarity_setup(runner):
    """--id_similarity's requirements; raises ValueError with the reason.  Returns the validated --id_weights state
    dict (arcface.load_state_dict)."""
    from .arcface import check_image_size, load_state_dict
    a = runner.args
    if getattr(a, "pass_editing", False):
        raise ValueError("--id_similarity scores the edited images: with --pass_editing nothing is edited")
    size = runner.config.data.image_size
    try:
        check_image_size(size, size)
    except ValueError as e:
        raise ValueError(f"--id_similarity: {e}") from None
    path = getattr(a, "id_weights", None)
    if not path or not os.path.isfile(path):
        raise ValueError(f"--id_similarity: --id_weights {path!r} is not a file (the reference's "
                         "pretrained/model_ir_se50.pth)")
    try:
        return load_state_dict(path)
    except ValueError as e:
        raise ValueError(f"--id_similarity: {e}") from None


def seg_consistency_setup(runner):
    """--seg_consistency's requirements; raises ValueError with the reason.  Returns the validated --seg_weights state
    dict (face_parsing.load_state_dict)."""
    a = runner.args
    if getattr(a, "pass_editing", False):
        raise ValueError("--seg_consistency scores the edited images: with --pass_editing nothing is edited")
    return seg_weights(runner, "--seg_consistency")


def seg_weights(runner, flag):
    """the validated --seg_weights state dict (face_parsing.load_state_dict) for `flag`; ValueError with the reason"""
    from .face_parsing import load_state_dict
    path = getattr(runner.args, "seg_weights", None)
    if not path or not os.path.isfile(path):
        raise ValueError(f"{flag}: --seg_weights {path!r} is not a file (a torch.save of the face-parsing "
                         "BiSeNet(n_classes=19) state dict, e.g. 79999_iter.pth)")
    try:
        return load_state_dict(path)
    except ValueError as e:
        raise ValueError(f"{flag}: {e}") from None


def content_preservation_setup(runner):
    """--content_preservation's requirements; raises ValueError with the reason.  Returns what ContentPreservation
    takes: the validated --lpips_weights path, or seeded weights with --synthetic_weights (as Asyrp.load_lpips)."""
    from .lpips import load_state_dict
    from .preservation import check_image_size
    a = runner.args
    if not getattr(a, "run_test", False) or getattr(a, "diff_style", False):
        raise ValueError("--content_preservation scores the edits of --run_test (not --diff_style or --lpips)")
    if getattr(a, "pass_editing", False):
        raise ValueError("--content_preservation scores the edited images: with --pass_editing nothing is edited")
    size = runner.config.data.image_size
    try:
        check_image_size(size, size)
    except ValueError as e:
        raise ValueError(f"--content_preservation: {e}") from None
    path = getattr(a, "lpips_weights", None)
    if path:
        if not os.path.isfile(path):
            raise ValueError(f"--content_preservation: --lpips_weights {path!r} is not a file")
        try:
            load_state_dict(path)
        except Exception as e:  # a file torch.load cannot read, or the wrong keys
            raise ValueError(f"--content_preservation: --lpips_weights {path!r}: {e}") from None
        return path
    if getattr(a, "synthetic_weights", False):
        from .synthetic import lpips_state_dict
        return lpips_state_dict(seed=getattr(a, "seed", 1234))
    raise ValueError("--content_preservation needs --lpips_weights (a torch.save of the lpips package's "
                     "LPIPS(net='alex').state_dict()) or --synthetic_weights")


def dino_structure_setup(runner):
    """--dino_structure's requirements; raises ValueError with the reason.  Returns the validated --dino_weights state
    dict (the tensors of dino.load_state_dict).  It scores the edits of --run_test and the results of --diff_style."""
    from .dino import load_state_dict
    a = runner.args
    if getattr(a, "pass_editing", False):
        raise ValueError("--dino_structure scores the edited images: with --pass_editing nothing is edited")
    if not (getattr(a, "run_test", False) or getattr(a, "diff_style", False)) or getattr(a, "lpips", False) or \
            getattr(a, "h_directions", False):
        raise ValueError("--dino_structure scores the edits of --run_test and the results of --diff_style (not --lpips "
                         "or --h_directions)")
    path = getattr(a, "dino_weights", None)
    if not path or not os.path.isfile(path):
        raise ValueError(f"--dino_structure: --dino_weights {path!r} is not a file (a torch.save of DINO's "
                         "VisionTransformer state dict, e.g. dino_vitbase8_pretrain.pth)")
    try:
        return load_state_dict(path)[1]
    except ValueError as e:
        raise ValueError(f"--dino_structure: {e}") from None


def fid_setup(runner):
    """--fid's requirements; raises ValueError with the reason.  Returns the validated --fid_weights state dict
    (fid.load_state_dict)."""
    from .fid import load_state_dict, validate_stats
    a = runner.args
    ref = getattr(a, "fid_ref", None)
    if ref is not None:  # the headers only; rank 0 reads the arrays in Scorers.finish
        if a.kid_subsets < 0 or a.kid_subset_size < 2:
            raise ValueError(f"--fid_ref: --kid_subsets must be >= 0 and --kid_subset_size >= 2, got "
                             f"{a.kid_subsets} and {a.kid_subset_size}")
        try:
            validate_stats(ref)
        except ValueError as e:
            raise ValueError(f"--fid_ref: {e}") from None
    if getattr(a, "pass_editing", False):
        raise ValueError("--fid scores the edited images: with --pass_editing nothing is edited")
    if getattr(a, "diff_style", False):
        raise ValueError("--fid scores the sets of --run_test; --diff_style is not scored")
    path = getattr(a, "fid_weights", None)
    if not path or not os.path.isfile(path):
        raise ValueError(f"--fid: --fid_weights {path!r} is not a file (pytorch-fid's "
                         "pt_inception-2015-12-05-6726825d.pth)")
    try:
        return load_state_dict(path)
    except ValueError as e:
        raise ValueError(f"--fid: {e}") from None


class Scorers:
    """The scores one --run_test asks for.  Construction runs their requirement checks (before any model loads);
    `with scorers:` builds their networks for the run and releases them, and the CUDA cache, at its end.
    attrs (an attribute sweep): tuple k is attribute k; directional CLIP scores each attribute's rows with its own
    texts, and every table names the attribute in an `attr` column."""

    def __init__(self, runner, attrs=None):
        a = runner.args
        self.runner, self.attrs = runner, attrs
        clip = runner.directional_clip_setup(attrs) if getattr(a, "DirectionalClipSmilarity", False) else None
        self.texts = clip[:2] if clip else None  # (source, target) text, or lists of one per attribute
        # what each network is built from, in the order the checks run and the networks are built
        specs = {"clip": clip[2] if clip else None,
                 "id": runner.id_similarity_setup() if getattr(a, "id_similarity", False) else None,
                 "seg": runner.seg_consistency_setup() if getattr(a, "seg_consistency", False) else None,
                 "fid": runner.fid_setup() if getattr(a, "fid", False) else None,
                 "cp": runner.content_preservation_setup() if getattr(a, "content_preservation", False) else None,
                 "dino": runner.dino_structure_setup() if getattr(a, "dino_structure", False) else None}
        self.specs = {name: spec for name, spec in specs.items() if spec is not None}
        self.needs_origin = bool(self.specs)  # every score compares against the origin pass
        # --content_preservation and --dino_structure of latents inverted from images also score the origin pass
        # against those images
        self.keeps_source = ("cp" in self.specs or "dino" in self.specs) and not a.load_random_noise
        self.nets = {}

    def __enter__(self):
        from .arcface import ArcFace
        from .clip_image import CLIPLoss
        from .face_parsing import FaceParser
        from .fid import FeatureSets, FIDInception
        from .dino import DINO
        from .preservation import ContentPreservation
        a, dev = self.runner.args, self.runner.device
        build = {"clip": lambda s: CLIPLoss(a.clip_weights, a.clip_vocab, s, device=dev),
                 "id": lambda s: ArcFace(s, device=dev), "seg": lambda s: FaceParser(s, device=dev),
                 "fid": lambda s: FIDInception(s, device=dev), "cp": lambda s: ContentPreservation(s, device=dev),
                 "dino": lambda s: DINO(s, device=dev)}
        try:
            for name in list(self.specs):  # the host copies of the weights go once their network is built
                self.nets[name] = build[name](self.specs.pop(name))
        except BaseException:
            self.__exit__()
            raise
        self.fid_sets = FeatureSets()  # the pool features --fid collects over the whole run
        return self

    def __exit__(self, *exc):
        if self.nets:  # the networks live for one run only
            self.nets = {}
            torch.cuda.empty_cache()

    def score(self, file_name, folder, mode, batch_ids, origin, edited, coeffs, x0_source=None):
        """the scores of one batch of save_image: every tuple's edits (edited[k], [images]) against the origin pass,
        written to <folder>/<file_name>_ngen<n_train_step>_<score>.tsv and kept in runner.<score>[file_name]; the
        --fid pool features added to their sets with the batch's image indices (batch_ids).  x0_source: the input
        images the latents were inverted from, which --content_preservation scores the origin pass against."""
        if not (edited and self.nets):  # without scores there is no origin pass to score against
            return
        r, nets = self.runner, self.nets
        bs, n = origin.shape[0], len(edited)
        stem = os.path.join(folder, f"{file_name}_ngen{r.args.n_train_step}_")

        def keep(name, scores, column, label, origin_rows=None):
            getattr(r, name)[file_name] = scores
            write_scores(f"{stem}{name}.tsv", coeffs, scores, column, label, attrs=self.attrs, origin=origin_rows)

        if "clip" in nets:
            src, trg = self.texts
            if self.attrs is None:  # one text pair for every tuple: one call over all of them
                s_dir = nets["clip"].directional_similarity(origin, src, torch.cat(edited), trg).view(n, bs)
            else:
                s_dir = torch.stack([nets["clip"].directional_similarity(origin, src[k], edited[k], trg[k]).view(bs)
                                     for k in range(n)])
            keep("directional_clip", s_dir, "S_dir", "directional CLIP similarity")
        if "id" in nets:
            keep("id_similarity", nets["id"].id_similarity(origin, torch.cat(edited)).view(n, bs), "ID",
                 "identity similarity")
        if "seg" in nets:
            keep("seg_consistency", nets["seg"].seg_consistency(origin, torch.cat(edited)).view(n, bs), "SC",
                 "segmentation consistency")
        if "fid" in nets:
            feats = nets["fid"].features(torch.cat([origin.cpu()] + [e.cpu() for e in edited]))
            self.fid_sets.add(mode, "origin", batch_ids, feats[:bs])
            for k in range(n):
                self.fid_sets.add(mode, k, batch_ids, feats[(k + 1) * bs:(k + 2) * bs])
        if "cp" in nets:
            from .preservation import COLUMNS
            cp = nets["cp"].scores(origin, torch.cat(edited)).view(n, bs, len(COLUMNS))
            rec = None
            if x0_source is not None:
                rec = r.reconstruction[file_name] = nets["cp"].scores(x0_source, origin)
            keep("content_preservation", cp, COLUMNS, "content preservation", rec)
        if "dino" in nets:
            sc = nets["dino"].scores(origin, torch.cat(edited))
            rec = None
            if x0_source is not None:
                rec = r.dino_origin[file_name] = nets["dino"].scores(x0_source, origin)[0]
            keep("dino", sc, DINO_COLUMNS, "DINO structure distance / CLS cosine", rec)

    def finish(self, coeffs):
        """--fid at the end of a run (finish_fid, through Asyrp.finish_fid).  Every rank must call it, also one that
        ran no batch."""
        if "fid" in self.nets:
            self.runner.finish_fid(self.fid_sets, coeffs, attrs=self.attrs)


def finish_fid(runner, sets, coeffs, attrs=None):
    """--fid at the end of a run: every rank's pool features (fid.FeatureSets) to rank 0, which sorts each set by image
    index and scores every tuple's edited set against the origin set of the same pass: printed, kept in
    runner.fid[mode] and written to <test_image_folder>/<mode>_ngen<n_train_step>_fid.tsv.  With --fid_ref also
    against the real images' statistics (_fid_real.tsv); with --prdc also precision / recall / density / coverage
    from the same features (_prdc.tsv, and _prdc_real.tsv against --fid_ref's features, whose radii are computed
    once)."""
    from .fid import fid_kid, knn_radii, load_stats, prdc, score_against_stats, set_moments
    a = runner.args
    pk = a.prdc_k if getattr(a, "prdc", False) else None
    dist_on = runner.world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized()
    got = sets.gather(runner.rank, runner.world if dist_on else 1)
    if got is None:
        return
    real = None
    if getattr(a, "fid_ref", None) is not None:  # --fid_ref: the real images' statistics, read once
        real = load_stats(a.fid_ref)
        if "features" in real:
            real["features"] = torch.from_numpy(real["features"]).to(runner.device)
    real_radii = None  # --prdc --fid_ref: the real images' k-NN radii, for every set of both passes
    if pk is not None and real is not None and real.get("features") is not None and real["features"].shape[0] > pk:
        real_radii = knn_radii(real["features"], pk)
    for mode in ("train", "test"):
        if (mode, "origin") not in got:
            continue
        ids, ref = got[(mode, "origin")]
        ref = ref.to(runner.device).contiguous()
        ref_moments = set_moments(ref) if ref.shape[0] >= 2 else None
        rows, edited = [], []
        for k in range(len(coeffs)):
            ids_k, feats = got[(mode, k)]
            if not torch.equal(ids_k, ids):
                raise RuntimeError(f"--fid: tuple {k} of the {mode} pass has other images than its origin set")
            edited.append(feats.to(runner.device).contiguous())
            rows.append(fid_kid(ref, edited[-1], ref_moments))
        runner.fid[mode] = torch.tensor(rows, dtype=torch.float64)
        os.makedirs(a.test_image_folder, exist_ok=True)
        stem = os.path.join(a.test_image_folder, f"{mode}_ngen{a.n_train_step}_")
        write_fid(stem + "fid.tsv", coeffs, rows, ref.shape[0], mode, attrs=attrs)
        if real is not None:
            real_rows = [score_against_stats(f, real, a.kid_subsets, a.kid_subset_size, m)
                         for f, m in [(ref, ref_moments)] + [(e, None) for e in edited]]
            runner.fid_real[mode] = torch.tensor(real_rows, dtype=torch.float64)
            n_ref = real["features"].shape[0] if "features" in real else None
            write_fid_real(stem + "fid_real.tsv", coeffs, real_rows, ref.shape[0], n_ref, mode, attrs=attrs)
        if pk is None:
            continue
        origin_radii = knn_radii(ref, pk) if ref.shape[0] > pk else None
        prdc_rows = [prdc(ref, e, pk, origin_radii) for e in edited]
        runner.prdc[mode] = torch.tensor(prdc_rows, dtype=torch.float64)
        write_prdc(stem + "prdc.tsv", coeffs, prdc_rows, ref.shape[0], None, mode, attrs=attrs)
        if real is not None:
            if "features" in real:
                prdc_rows = [prdc(real["features"], f, pk, real_radii) for f in [ref] + edited]
                n_ref = real["features"].shape[0]
            else:
                prdc_rows, n_ref = [(math.nan,) * 4] * (1 + len(edited)), None
            runner.prdc_real[mode] = torch.tensor(prdc_rows, dtype=torch.float64)
            write_prdc(stem + "prdc_real.tsv", coeffs, prdc_rows, ref.shape[0], n_ref, mode, attrs=attrs,
                       real=True)


# ---------------------------------------------------------------------------------------------------------------------
# score tables
# ---------------------------------------------------------------------------------------------------------------------
def _coeff_text(tup):
    """an hs_coeff tuple as the tables write it: 1,0.5"""
    return ",".join(f"{float(c):.6g}" for c in tup)


def _tuple_name(coeffs, attrs, k):
    """tuple k as the printed lines name it: attribute <attr> under a sweep, else hs_coeff (1.0, 0.5)"""
    return f"attribute {attrs[k]}" if attrs is not None else f"hs_coeff {tuple(float(c) for c in coeffs[k])}"


DINO_COLUMNS = ("structure", "cls_cos")
DIFF_STYLE_DINO_COLUMNS = ("content", "style", "hs_coeff", "structure_content", "structure_style", "cls_cos_content",
                           "cls_cos_style")


def write_diff_style_dino(path, rows):
    """--diff_style --dino_structure's table: rows (content path, style path, γ, structure_content, structure_style,
    cls_cos_content, cls_cos_style), sorted by (content, style, γ), so that the file does not depend on how the rows
    were chunked or sharded; prints each row"""
    rows = sorted(rows, key=lambda r: (r[0], r[1], float(r[2])))
    with open(path, "w") as f:
        f.write("\t".join(DIFF_STYLE_DINO_COLUMNS) + "\n")
        for c, s_, g, *vals in rows:
            f.write("\t".join([c, s_, f"{float(g):.6g}"] + [repr(float(v)) for v in vals]) + "\n")
    for c, s_, g, sc, ss, cc, cs in rows:
        print(f"DINO, content {c}, style {s_}, hs_coeff {float(g):.6g}: structure against the content {sc:.6f}, "
              f"against the style {ss:.6f}; CLS cosine with the content {cc:.6f}, with the style {cs:.6f}")
    return rows


def gather_rows(runner, rows):
    """every rank's list of rows to rank 0 (torch.distributed.gather_object, as fid.FeatureSets.gather does): the
    concatenation on rank 0, None on the other ranks; the list itself without a process group"""
    dist_on = runner.world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized()
    if not dist_on:
        return list(rows)
    got = [None] * runner.world if runner.rank == 0 else None
    torch.distributed.gather_object(list(rows), got, dst=0)
    return None if runner.rank != 0 else [r for part in got for r in part]


def write_scores(path, coeffs, scores, column, label, attrs=None, origin=None):
    """a per-edit score table: one row per (hs_coeff tuple, image) in grid order, columns image, tuple, hs_coeff and
    `column`; prints each tuple's mean as `label`.  attrs (an attribute sweep): tuple k is attribute k, named in an
    appended `attr` column.  Several columns: `column` a sequence of names and scores [tuples][images][columns].
    origin ([images][columns]): rows of the origin pass first, with tuple `origin`, hs_coeff `-` (and attr `-`)"""
    columns = [column] if isinstance(column, str) else list(column)
    tail = (lambda a: f"\t{a}") if attrs is not None else (lambda a: "")

    def cells(v):
        return "\t".join(repr(x) for x in (v if isinstance(v, list) else [v]))
    with open(path, "w") as f:
        f.write("image\ttuple\ths_coeff\t" + "\t".join(columns) + tail("attr") + "\n")
        if origin is not None:
            for i, v in enumerate(origin.tolist()):
                f.write(f"{i}\torigin\t-\t{cells(v)}" + tail("-") + "\n")
        for k, row in enumerate(scores.tolist()):
            tup = _coeff_text(coeffs[k])
            for i, v in enumerate(row):
                f.write(f"{i}\t{k}\t{tup}\t{cells(v)}" + tail(attrs[k] if attrs is not None else None) + "\n")
    rows = ([("origin", origin)] if origin is not None else []) + [
        (_tuple_name(coeffs, attrs, k), row) for k, row in enumerate(scores)]
    for name, row in rows:
        means = row.double().reshape(row.shape[0], -1).mean(0).tolist()
        vals = f"{means[0]:.6f}" if len(columns) == 1 else ", ".join(f"{c} {m:.6f}" for c, m in zip(columns, means))
        print(f"{label}, {name}: mean {vals} over {row.shape[0]} images")


def _write_set_table(path, coeffs, rows, n, columns, attrs, real, n_ref=None):
    """a per-set table (write_fid / write_fid_real / write_prdc): one row per hs_coeff tuple, columns tuple, hs_coeff,
    n (images per set), `columns` (each value's repr as a float), and `attr` under an attribute sweep.  real (against
    real images' statistics): rows[0] is the origin set (tuple `origin`, hs_coeff `-`, attr `-`), and an n_ref column
    (reference images; `-` for a file without features) follows n.  Returns (tuple index or None for the origin set,
    hs_coeff text, values) of each row."""
    keys = ([(None, "origin", "-", "-")] if real else []) + [
        (k, str(k), _coeff_text(c), attrs[k] if attrs is not None else None) for k, c in enumerate(coeffs)]
    head = ["tuple", "hs_coeff", "n"] + ["n_ref"] * real + list(columns) + ["attr"] * (attrs is not None)
    with open(path, "w") as f:
        f.write("\t".join(head) + "\n")
        for (_, key, tup, attr), vals in zip(keys, rows):
            f.write("\t".join([key, tup, str(n)] + [_n_ref(n_ref)] * real + [repr(float(v)) for v in vals] +
                              [attr] * (attrs is not None)) + "\n")
    return [(k, tup, vals) for (k, _, tup, _), vals in zip(keys, rows)]


def _n_ref(n_ref):
    return "-" if n_ref is None else str(n_ref)


def write_fid(path, coeffs, rows, n, mode, attrs=None):
    """the FID / KID table of one pass: one row per hs_coeff tuple, columns tuple, hs_coeff, n (images per set), FID and
    KID (`attr` appended under an attribute sweep); prints each tuple's values"""
    for k, _, (fd, kd) in _write_set_table(path, coeffs, rows, n, ["FID", "KID"], attrs, False):
        print(f"FID / KID ({mode}, {n} images), {_tuple_name(coeffs, attrs, k)}: FID {fd:.6f}, KID {kd:.6f}")


def write_fid_real(path, coeffs, rows, n, n_ref, mode, attrs=None):
    """the table of one pass against real images' statistics (--fid_ref): rows[0] the origin set, rows[1 + k] tuple k's
    set, each (FID, KID, KID_mean, KID_std), with the n_ref column; values as write_fid writes them.  Prints each
    row's values"""
    for k, _, (fd, kd, km, ks) in _write_set_table(path, coeffs, rows, n, ["FID", "KID", "KID_mean", "KID_std"], attrs,
                                                   True, n_ref):
        name = "origin" if k is None else _tuple_name(coeffs, attrs, k)
        print(f"FID / KID against the real images ({mode}, {n} images, {_n_ref(n_ref)} reference), {name}: "
              f"FID {fd:.6f}, KID {kd:.6f}, subset KID {km:.6f} +- {ks:.6f}")


def write_prdc(path, coeffs, rows, n, n_ref, mode, attrs=None, real=False):
    """the precision / recall / density / coverage table of one pass (--prdc): one row per hs_coeff tuple, values as
    write_fid writes them.  real (--fid_ref): rows[0] is the origin set, with the n_ref column.  Prints each row"""
    against = f"against the real images ({mode}, {n} images, {_n_ref(n_ref)} reference)" if real else \
        f"({mode}, {n} images)"
    for k, tup, (p, rc, d, c) in _write_set_table(path, coeffs, rows, n, ["precision", "recall", "density", "coverage"],
                                                  attrs, real, n_ref):
        name = "origin" if k is None else (f"attribute {attrs[k]}" if attrs is not None else f"hs_coeff ({tup})")
        print(f"precision / recall / density / coverage {against}, {name}: P {p:.6f}, R {rc:.6f}, D {d:.6f}, "
              f"C {c:.6f}")
