"""`Asyrp` runner — inference/editing half of the reference's diffusion_latent.py on the CUDA engine.

Mirrors, with the same attribute / flag names:
  Asyrp.__init__               diffusion_latent.py:32-73    betas, logvar tables
  Asyrp.load_pretrained_model  :76-126                      dataset -> UNet family dispatch, load_state_dict(strict=False)
  Asyrp.run_test               :547-874                     sequences, Δh checkpoint, hs_coeff (single / multi-attribute /
                                                            interpolation sweep), batching of latents
  Asyrp.save_image             :445-544                     the reverse loops + PNG grid; with --attr_sweep one row
                                                            schedule per attribute (run_attr_sweep)
  Asyrp.random_noise_pairs     :1087-1188                   x_T = N(0,1) per image
  Asyrp.set_t_edit_t_addnoise  :1308-1416                   user-defined values or LPIPS-table lookup given a cosine
                                                            (--clip_cosine, or CLIP's text cosine on the GPU)
  Asyrp.compute_lpips_distance :1191-1303                   --lpips: the LPIPS(x_t, x0) / LPIPS(x0_t, x0) tables of an
                                                            inversion, which set_t_edit_t_addnoise reads
  scoring.Scorers              main.py:101, losses/*.py     the edit scores of run_test and run_attr_sweep: each edit
                                                            against the origin pass of the same x_T, written next to
                                                            the PNG, and the sets of edits at the end of the run:
    --DirectionalClipSmilarity                              CLIPLoss's directional similarity (clip_image.CLIPLoss)
    --id_similarity                                         1 - IDLoss (ArcFace IR-SE50, arcface.ArcFace); the
                                                            reference uses IDLoss only in training
    --seg_consistency                                       segmentation consistency of a face-parsing BiSeNet
                                                            (face_parsing.FaceParser); this build's definition
    --content_preservation                                  PSNR, SSIM, MS-SSIM and LPIPS-Alex
                                                            (preservation.ContentPreservation), and the origin pass
                                                            against the input image for inverted latents; this
                                                            build's definition
    --dino_structure                                        DINO-ViT key self-similarity structure distance and CLS
                                                            cosine (dino.DINO), with the same origin rows; also each
                                                            --diff_style result against its content and its style
    --fid                                                   FID and KID of each set of edits (one per hs_coeff tuple)
                                                            against the origin pass on Inception-v3 pool features
                                                            (fid.FIDInception), gathered to rank 0 at the end of the
                                                            run; this build's definition; with --fid_ref also against
                                                            real images' statistics (fid.score_against_stats); with
                                                            --prdc also precision / recall / density / coverage
                                                            (fid.prdc)
  Asyrp.precompute_pairs_with_h :877-947                    DDIM inversion of one image keeping the bottleneck h of
                                                            every step (batched here, same cache file)
  Asyrp.run_diff_style         main.py:192-202              --diff_style (DiffStyle content injection): this build's
                                                            composition of the functions above with denoising_step's
                                                            delta_h branch; the reference declares the flags only
  Asyrp.run_h_directions       (none)                       --h_directions: editing directions from the statistics of
                                                            the bottleneck h (hspace.py), applied by --run_test
                                                            --h_direction as h + α d; this build's definition
  Asyrp.run_region_compose     (none)                       --region_compose: several attributes composed into one
                                                            image, each in its own face-parsing region, inside the
                                                            per-row trajectory; this build's definition

Differences (documented in INTEGRATION.md): the reverse loop is UNetEngine.sample() — one CUDA graph per
(batch, schedule) instead of 40 Python iterations; pretrained weights come from --model_path (no URL download);
the CLIP text cosine that picks t_edit runs on this library's kernels (clip_text.CLIPText) from --clip_weights and
--clip_vocab, or is given as --clip_cosine; SRC_TRG_TXT_DIC is read from --text_dic (default utils/text_dic.py).
With torch.distributed initialised (one process per GPU) the image batches are sharded round-robin across ranks;
the collectives are the initial weight broadcast and, with --fid, the end-of-run gather of the pool features to rank
0; each rank computes the CLIP cosine itself (the kernels are deterministic, so every rank picks the same t_edit).
"""
import ast
import os
import time

import numpy as np
import torch

from . import scoring
from .modules import DDPM, guided_Diffusion, i_DDPM
from .schedule import RowSchedule, Schedule, make_sequences
from .scoring import write_fid, write_fid_real, write_prdc, write_scores  # noqa: F401  (the tables' former home)
from .utils.diffusion_utils import get_beta_schedule


class Asyrp(object):
    def __init__(self, args, config, device=None):
        self.args = args
        self.config = config
        if device is None:
            device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
        self.device = torch.device(device)
        self.model_var_type = config.model.var_type
        betas = get_beta_schedule(beta_start=config.diffusion.beta_start, beta_end=config.diffusion.beta_end,
                                  num_diffusion_timesteps=config.diffusion.num_diffusion_timesteps)
        self.betas = torch.from_numpy(betas).float().to(self.device)
        self.num_timesteps = betas.shape[0]
        alphas = 1.0 - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        alphas_cumprod_prev = np.append(1.0, alphas_cumprod[:-1])
        posterior_variance = betas * (1.0 - alphas_cumprod_prev) / (1.0 - alphas_cumprod)
        self.alphas_cumprod = alphas_cumprod
        if self.model_var_type == "fixedlarge":
            self.logvar = np.log(np.append(posterior_variance[1], betas[1:]))
        elif self.model_var_type == 'fixedsmall':
            self.logvar = np.log(np.maximum(posterior_variance, 1e-20))
        self.learn_sigma = False  # set by load_pretrained_model()
        self.t_edit = getattr(args, "user_defined_t_edit", None)
        self.t_addnoise = getattr(args, "user_defined_t_addnoise", None)
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.directional_clip = {}  # --DirectionalClipSmilarity: save_image's file name -> S_dir [tuples][images]
        self.id_similarity = {}  # --id_similarity: save_image's file name -> 1 - IDLoss [tuples][images]
        self.seg_consistency = {}  # --seg_consistency: save_image's file name -> SC [tuples][images]
        self.fid = {}  # --fid (rank 0): 'train' / 'test' -> fp64 [tuples][2], (FID, KID) of each tuple's set
        # --fid_ref (rank 0): 'train' / 'test' -> fp64 [1 + tuples][4], (FID, KID, KID_mean, KID_std) against the real
        # images' statistics of the origin set (row 0) and of each tuple's set
        self.fid_real = {}
        # --prdc (rank 0): 'train' / 'test' -> fp64 [tuples][4], (precision, recall, density, coverage) of each tuple's
        # set against the origin set; with --fid_ref, prdc_real: fp64 [1 + tuples][4] against the real images' features
        self.prdc = {}
        self.prdc_real = {}
        # --content_preservation: save_image's file name -> fp64 [tuples][images][4], (PSNR, SSIM, MS_SSIM, LPIPS) of
        # each edit against the origin pass; reconstruction: fp64 [images][4] of the origin pass against the input
        # image, for latents inverted from images
        self.content_preservation = {}
        self.reconstruction = {}
        # --dino_structure: save_image's file name -> fp64 [tuples][images][2], (structure distance, CLS cosine) of each
        # edit against the origin pass; dino_origin: fp64 [images][2] of the origin pass against the input image, for
        # latents inverted from images; diff_style_dino (rank 0): the sorted rows of --diff_style's table
        self.dino = {}
        self.dino_origin = {}
        self.diff_style_dino = None

    # ------------------------------------------------------------------------------------------
    def load_pretrained_model(self):
        ds = self.config.data.dataset
        if ds in ["CelebA_HQ", "LSUN", "CelebA_HQ_Dialog", "CUSTOM"]:
            model = DDPM(self.config)
            self.learn_sigma = False
        elif ds in ["FFHQ", "AFHQ", "IMAGENET"]:
            model = i_DDPM(ds)
            self.learn_sigma = True
        elif ds in ["MetFACE", "CelebA_HQ_P2"]:
            model = guided_Diffusion(ds)
            self.learn_sigma = True
        else:
            raise ValueError(f'Not implemented dataset {ds}')
        path = getattr(self.args, "model_path", None)
        if path:
            ckpt = torch.load(path, map_location="cpu", weights_only=True)
            model.load_state_dict(ckpt, strict=False)
        elif getattr(self.args, "synthetic_weights", False):
            from .synthetic import randomize_
            randomize_(model, seed=getattr(self.args, "seed", 1234))
        else:
            raise FileNotFoundError("no --model_path given: pretrained UNet weights cannot be downloaded here "
                                    "(pass --model_path <state dict> or --synthetic_weights)")
        return model

    # ------------------------------------------------------------------------------------------
    def set_t_edit_t_addnoise(self, LPIPS_th=0.33, LPIPS_addnoise_th=0.1, return_clip_loss=False, cosine=None):
        """t_edit = first t with LPIPS(x0_t, x0) >= LPIPS_th * cosine; t_addnoise = first t with LPIPS >= LPIPS_addnoise_th
        on the x_t table (--add_noise_from_xt) or the same x0_t table (diffusion_latent.py:1331-1410).  Each of
        --user_defined_t_edit / --user_defined_t_addnoise overrides its value.  The cosine is CLIP's text-direction
        similarity in the reference (:1319-1329): the `cosine` argument, else --clip_cosine, else, when t_edit is
        needed, CLIPText on --clip_weights / --clip_vocab with the texts of --edit_attr (or --src_txts / --trg_txts).
        Tables: <lpips_table_dir>/<config stem>_LPIPS_distance_{x0_t,x}.tsv (the reference ships them under utils/)."""
        a = self.args
        ut, ua = getattr(a, "user_defined_t_edit", None), getattr(a, "user_defined_t_addnoise", None)
        if ut is not None and ua is not None:
            self.t_edit, self.t_addnoise = ut, ua
            return cosine if cosine is not None else getattr(a, "clip_cosine", None)
        cosine = cosine if cosine is not None else getattr(a, "clip_cosine", None)
        tdir = getattr(a, "lpips_table_dir", None) or "utils"
        name = str(getattr(a, "config", "") or "").split(".")[0] or self.config.data.category
        name = os.path.basename(name)
        if name == "custom":
            name = getattr(a, "custom_dataset_name", "celeba")
        p0 = os.path.join(tdir, f"{name}_LPIPS_distance_x0_t.tsv")
        if not os.path.exists(p0) or (ut is None and cosine is None and not self.clip_configured()):
            raise ValueError(f"t_edit / t_addnoise undefined: pass --user_defined_t_edit and --user_defined_t_addnoise, "
                             f"or --clip_cosine, or --clip_weights and --clip_vocab, with --lpips_table_dir (looked "
                             f"for {p0})")
        if ut is None and cosine is None:
            cosine = self.clip_cosines([self.edit_texts()])[0]
        table = _read_tsv(p0)
        self.t_edit = ut if ut is not None else next(t for t, v in table if v >= LPIPS_th * cosine)
        if ua is not None:
            self.t_addnoise = ua
        else:
            if getattr(a, "add_noise_from_xt", False):
                table = _read_tsv(os.path.join(tdir, f"{name}_LPIPS_distance_x.tsv"))
            self.t_addnoise = next(t for t, v in table if v >= LPIPS_addnoise_th)
        return cosine

    def clip_configured(self):
        return bool(getattr(self.args, "clip_weights", None)) and bool(getattr(self.args, "clip_vocab", None))

    def needs_clip(self):
        """t_edit must come from CLIP's text cosine: no --user_defined_t_edit, no --clip_cosine"""
        a = self.args
        return getattr(a, "user_defined_t_edit", None) is None and getattr(a, "clip_cosine", None) is None

    def text_dic(self):
        return read_text_dic(getattr(self.args, "text_dic", None) or os.path.join("utils", "text_dic.py"))

    def edit_texts(self, attr=None):
        """(src_txts, trg_txts) of an attribute as the reference's __init__ picks them (:66-73): --src_txts /
        --trg_txts for --edit_attr None, SRC_TRG_TXT_DIC[attr] otherwise; the dictionary is read only here"""
        a = self.args
        attr = attr if attr is not None else getattr(a, "edit_attr", None)
        if attr is None:
            src, trg = getattr(a, "src_txts", None), getattr(a, "trg_txts", None)
            if not src or not trg:
                raise ValueError("--edit_attr None needs --src_txts and --trg_txts")
            return list(src), list(trg)
        if attr == "attribute":
            raise ValueError("--edit_attr attribute has no texts: CLIP's cosine needs --multiple_attr, an attribute "
                             "of SRC_TRG_TXT_DIC or --src_txts / --trg_txts")
        dic = self.text_dic()
        if attr not in dic:
            raise ValueError(f"attribute {attr!r} is not in SRC_TRG_TXT_DIC")
        return list(dic[attr][0]), list(dic[attr][1])

    # The score checks and the end of a --fid run live in scoring.py.  The runner keeps their names, and
    # scoring.Scorers calls them through it, so that a caller who replaces one on the runner replaces it for the run.
    def directional_clip_setup(self, attrs=None):
        return scoring.directional_clip_setup(self, attrs)

    def id_similarity_setup(self):
        return scoring.id_similarity_setup(self)

    def seg_consistency_setup(self):
        return scoring.seg_consistency_setup(self)

    def fid_setup(self):
        return scoring.fid_setup(self)

    def content_preservation_setup(self):
        return scoring.content_preservation_setup(self)

    def dino_structure_setup(self):
        return scoring.dino_structure_setup(self)

    def prdc_check(self):
        return scoring.prdc_check(self)

    def finish_fid(self, sets, coeffs, attrs=None):
        return scoring.finish_fid(self, sets, coeffs, attrs)

    @torch.no_grad()
    def clip_cosines(self, pairs):
        """CLIP's text-direction cosine of each (src_txts, trg_txts) pair (:1319-1329), printed as the reference
        prints it.  Each pair must hold one text per side (the reference takes .item()).  The encoder is built here
        and dropped before returning, so its buffers are gone before the UNet is loaded."""
        from .clip_text import CLIPText
        a = self.args
        clip = CLIPText(a.clip_weights, a.clip_vocab, device=self.device)
        try:
            out = []
            for src, trg in pairs:
                print("Texts:", src, trg)
                cos = clip.text_cosine(src, trg)
                if cos.numel() != 1:
                    raise ValueError(f"CLIP's cosine takes one source and one target text, got {src} and {trg}")
                print("text_cos_distance", cos.item())
                out.append(cos.item())
        finally:
            del clip
            torch.cuda.empty_cache()
        return out

    def choose_attribute(self, attrs):
        """--multiple_attr (:640-652): the attribute of the largest CLIP cosine (the first on a tie); sets
        src_txts / trg_txts to its texts and returns its cosine"""
        texts = [self.edit_texts(attr) for attr in attrs]
        cosines = self.clip_cosines(texts)
        best = max(range(len(attrs)), key=lambda i: (cosines[i], -i))
        print(f"Max cosine: {cosines[best]}, Max attribute: {attrs[best]}")
        self.src_txts, self.trg_txts = texts[best]
        return cosines[best]

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def random_noise_pairs(self, model=None, saved_noise=False, save_imgs=False):
        """[x0, x_rec, x_T] triples with x_T ~ N(0,1) drawn per image on the host (same draw order as :1172-1184).
        saved_noise (--saved_random_noise, :1099-1167): the latents and the images generated from them with the plain
        n_inv_step-step reverse process are cached as precomputed/<category>_<mode>_random_noise_nim<N>_ninv<k>_pairs.pth
        ([x_gen, x_gen, x_T] per image) and reused by later runs."""
        c, s = self.config.data.channels, self.config.data.image_size
        a = self.args
        out = {}
        if not saved_noise:
            for mode, n in (("train", a.n_train_img), ("test", a.n_test_img)):
                pairs = []
                for _ in range(n):
                    lat = torch.randn((1, c, s, s))
                    pairs.append([torch.zeros_like(lat), torch.zeros_like(lat), lat])
                out[mode] = pairs
            return out
        if self.config.data.dataset == "IMAGENET":
            raise NotImplementedError("--saved_random_noise with the IMAGENET class-conditional naming (:1103-1109)")
        seq_inv = [int(v + 1e-6) for v in list(np.linspace(0, 1, a.n_inv_step) * a.t_0)]
        seq_inv_next = [-1] + list(seq_inv[:-1])
        os.makedirs('precomputed', exist_ok=True)
        for mode, n in (("train", a.n_train_img), ("test", a.n_test_img)):
            p = os.path.join('precomputed/', f'{self.config.data.category}_{mode}_random_noise_nim{n}_ninv{a.n_inv_step}_pairs.pth')
            if os.path.exists(p):
                out[mode] = torch.load(p, map_location="cpu", weights_only=True)
                continue
            pairs = None
            if self.rank == 0:
                sch = Schedule(self.betas, seq_inv, seq_inv_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False,
                               sample_type=a.sample_type, logvars=self.logvar)
                pairs = []
                for _ in range(n):
                    lat = torch.randn((1, c, s, s))
                    x = self.edit_batch(model, lat, sch)
                    pairs.append([x.clone(), x.clone(), lat])
                _atomic_save(pairs, p)
            out[mode] = self._sync_cache(p, pairs)
        return out

    def _sync_cache(self, path, value):
        """rank 0 wrote `path`; the other ranks wait for it and load it"""
        if self.world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.barrier()
            if value is None:
                value = torch.load(path, map_location="cpu", weights_only=True)
        return value

    @torch.no_grad()
    def invert_batch(self, model, x0, n_inv_step=None, reconstruct=True):
        """DDIM inversion x_0 -> x_T followed by the reconstruction x_T -> x_rec with --sample_type, both as graph
        replays (precompute_pairs, diffusion_latent.py:1028-1072).  Returns (x_T, x_rec) on the host; x_rec is None
        without reconstruct."""
        a = self.args
        n = n_inv_step or a.n_inv_step
        seq_inv = [int(s + 1e-6) for s in list(np.linspace(0, 1, n) * a.t_0)]
        seq_inv_next = [-1] + list(seq_inv[:-1])
        eng = model.engine
        x_lat = eng.sample(x0.to(eng.device), Schedule.inversion(self.betas, seq_inv, seq_inv_next))
        if not reconstruct:
            return x_lat.cpu(), None
        sch = Schedule(self.betas, seq_inv, seq_inv_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False,
                       sample_type=getattr(a, "sample_type", "ddim"), logvars=self.logvar)
        noise = torch.randn((sch.n_stochastic, *x_lat.shape), device=eng.device) if sch.n_stochastic else None
        x_rec = eng.sample(x_lat, sch, noise=noise)
        return x_lat.cpu(), x_rec.cpu()

    @torch.no_grad()
    def precompute_pairs(self, model, save_imgs=False, modes=("train", "test")):
        """[x0, x_rec, x_T] triples per image, cached as precomputed/<category>_<mode>_t<t_0>_nim<N>_ninv<k>_pairs.pth
        — the reference's file name and list-of-triples format (:974-982,1072,1082).  Images come from
        --custom_train_dataset_dir / --custom_test_dataset_dir (png/jpg, resized to image_size, scaled to [-1, 1]);
        the reference's LMDB dataset classes are out of scope.  Under torchrun rank 0 inverts and writes the cache
        (temp file + rename), the other ranks load it after a barrier.  modes: the sets to return (--h_directions
        needs only "train")."""
        a, out = self.args, {}
        os.makedirs('precomputed', exist_ok=True)
        for mode, n in (("train", a.n_train_img), ("test", a.n_test_img)):
            if mode not in modes:
                continue
            p = os.path.join('precomputed/', f'{self.config.data.category}_{mode}_t{a.t_0}_nim{n}_ninv{a.n_inv_step}_pairs.pth')
            if os.path.exists(p) and not getattr(a, "re_precompute", False):
                out[mode] = torch.load(p, map_location="cpu", weights_only=True)
                continue
            pairs = None
            if self.rank == 0:
                folder = getattr(a, f"custom_{mode}_dataset_dir", None)
                if not folder or not os.path.isdir(folder):
                    raise FileNotFoundError(f"{p} not found and --custom_{mode}_dataset_dir is not a directory: nothing "
                                            "to invert (use --load_random_noise for random latents)")
                imgs = _load_image_folder(folder, self.config.data.image_size, n)
                pairs = []
                bs = max(1, a.bs_train)
                for k in range(0, len(imgs), bs):
                    x0 = torch.cat(imgs[k:k + bs], dim=0)
                    x_lat, x_rec = self.invert_batch(model, x0)
                    for i in range(x0.shape[0]):
                        pairs.append([x0[i:i + 1].clone(), x_rec[i:i + 1].clone(), x_lat[i:i + 1].clone()])
                _atomic_save(pairs, p)
            out[mode] = self._sync_cache(p, pairs)
        return out

    # ------------------------------------------------------------------------------------------
    def make_schedule(self, seq, seq_next, hs_coeff, edit=True, addnoise=True):
        """what save_image passes to denoising_step on every step (:476-483 origin pass, :507-520 edit pass): the
        origin pass gets neither dt_lambda nor ignore_timestep"""
        a = self.args
        return Schedule(self.betas, seq, seq_next, t_edit=self.t_edit, t_addnoise=self.t_addnoise if addnoise else 0,
                        hs_coeff=hs_coeff, edit=edit, sample_type=getattr(a, "sample_type", "ddim"),
                        dt_lambda=getattr(a, "dt_lambda", 1.0) if edit else 1.0, dt_end=999,
                        ignore_timestep=bool(getattr(a, "ignore_timesteps", False)) if edit else False,
                        logvars=self.logvar)

    @torch.no_grad()
    def edit_batch(self, model, x_lat, schedule, noise=None, out=None, **sample_kw):
        """x_T (host or device, [B,3,S,S]) -> edited x_0 on the host.  One graph replay; the H2D copy of x_T and the
        D2H copy of x_0 are the only transfers.  The N(0,1) draws of the stochastic steps are made on the device
        up-front, as the reference's torch.randn_like does per step (utils/diffusion_utils.py:79,97), unless `noise`
        ([n_stochastic, B, 3, S, S]) is given.  sample_kw: delta_hs / use_mask / record_dh / record_process / hs_coeffs
        of UNetEngine.sample(); hs_coeffs ([B][1 + n_delta] fp32) gives every row its own hs_coeff tuple, so one batch
        can mix attributes or edit strengths."""
        eng = model.engine
        dev = eng.device
        if schedule.n_stochastic and noise is None and sample_kw.get("anchors") is None:  # anchored: no noise
            noise = torch.randn((schedule.n_stochastic, *x_lat.shape), device=dev)
        elif noise is not None:
            noise = noise.to(dev, non_blocking=True)
        x0 = eng.sample(x_lat.to(dev, non_blocking=True), schedule, noise=noise, **sample_kw)
        if out is not None:
            out.copy_(x0, non_blocking=True)
            return out
        return x0.cpu()

    def _write_process(self, eng, schedule, folder, prefix, bs, rows=slice(None)):
        """per-step grids of [x_t ; x0_t] (save_process_origin / save_process_delta_h, :485-491,523-527) of the batch
        rows `rows` of the last replay"""
        import torchvision.utils as tvu
        rec = eng.last_records
        os.makedirs(folder, exist_ok=True)
        for k, st in enumerate(schedule.steps):
            out = (torch.cat([rec["x"][k][rows], rec["x0_t"][k][rows]], dim=0).cpu() + 1) * 0.5
            tvu.save_image(tvu.make_grid(out, nrow=bs, padding=1), os.path.join(folder, f'{prefix}_{int(st.t)}.png'))

    @torch.no_grad()
    def save_image(self, model, x_lat_tensor, seq_inv, seq_inv_next, save_x0=False, save_x_origin=False,
                   save_process_delta_h=False, save_process_origin=False, x0_tensor=None, delta_h_dict=None,
                   get_delta_hs=False, folder_dir="", file_name="", hs_coeff=(1.0, 1.0), h_direction=None,
                   sweep_times=None, scorers=None, mode=None, batch_ids=None, x0_source=None, edit_region=None,
                   region_compose=None, anchors=None):
        """rows of the grid: [x0] [origin DDIM] one row per hs_coeff tuple  (diffusion_latent.py:445-544).

        delta_h_dict: {t: None | Δh tensor}.  Entries that are tensors select the explicit-Δh branch for that step
        (raw-Δh checkpoints, mean Δh); get_delta_hs: run the DeltaBlocks and ADD their per-step output into
        delta_h_dict (mean-Δh extraction, :528-532).
        h_direction: a direction file (hspace.load_direction) for --h_direction: each tuple is (c0, α) and its rows take
        h2 = c0 h + α d_t at every edit step, every tuple a row block of one batch as for DeltaBlocks.
        sweep_times (--attr_sweep): tuple k is attribute k, its rows run with its own (t_edit, t_addnoise)
        sweep_times[k] (sweep_schedule); rows (attribute, image), attribute-major, in chunks of whole attributes of at
        most --max_rows_per_replay rows.
        scorers: a scoring.Scorers, which scores every tuple's edits against the origin pass of the same x_T (run for
        this even without save_x_origin, then left out of the grid); mode, batch_ids (the image index of every row)
        and x0_source (the input images the latents were inverted from) are passed on to Scorers.score.
        edit_region (--edit_region): (FaceParser, class indices, dilate r, feather sigma).  The origin pass then records
        x_t after every step and always runs; its x0 is parsed into one soft mask per image (region.region_masks),
        written as <file>_ngen<n>_region_mask.png, and every step of the edit pass ends with x <- m x + (1 - m) x_orig
        (UNetEngine.sample's blend), so that outside the region the edits follow the origin pass.
        region_compose (--region_compose): (FaceParser, class indices per attribute, r, sigma, (t_edit, t_addnoise) per
        attribute, coefficients per attribute).  As with edit_region the origin pass records its trajectory and always
        runs; its x0 gives K masks per image (region.compose_masks), written as <file>_ngen<n>_region_compose.png
        (one row per attribute), and hs_coeff is the one tuple the composite is scored as.  The grid's last row is the
        composite of every image (compose_batch).
        anchors (--exact_inversion): the inversion.Anchors of the batch's input images (anchor_batch), x_lat_tensor
        their x_T.  No origin pass runs: the origin is the input image, which an unedited anchored pass returns bit for
        bit.  Every edit pass is anchored (UNetEngine.sample's anchors, no noise drawn), and the region masks parse the
        input image and blend against the anchors' trajectory A[1:]."""
        import torchvision.utils as tvu
        a = self.args
        time_s = time.time()
        eng = model.engine
        bs = x_lat_tensor.shape[0]
        x_list, origin = [], None
        if save_x0 and x0_tensor is not None:
            x_list.append(x0_tensor.cpu())
        blend = None
        masked = edit_region is not None or region_compose is not None  # the edits follow the recorded origin pass
        kw_a = {"anchors": anchors} if anchors is not None else {}
        if anchors is not None and (save_x_origin or (scorers is not None and scorers.needs_origin) or masked):
            origin = anchors.x0.cpu()  # the anchored origin pass: the input image, exactly
            if save_x_origin:
                x_list.append(origin)
        elif save_x_origin or (scorers is not None and scorers.needs_origin) or masked:
            sch = self.make_schedule(seq_inv, seq_inv_next, (1.0,), edit=False,
                                     addnoise=bool(getattr(a, "origin_process_addnoise", False)))
            if save_x_origin:
                origin = self.edit_batch(model, x_lat_tensor, sch, record_process=save_process_origin or masked)
                x_list.append(origin)
                if save_process_origin:
                    self._write_process(eng, sch, os.path.join(folder_dir, file_name), "origin", bs)
            else:  # the pass only the score needs leaves the random stream as it was: the edits draw the same noise
                with torch.random.fork_rng(devices=[eng.device]):
                    origin = self.edit_batch(model, x_lat_tensor, sch, record_process=masked)
        if masked:
            # the origin pass's trajectory; anchored, the inversion's (the anchors are copies the replays do not reuse)
            ref = anchors.ref if anchors is not None else eng.last_records["x"].clone()
            if edit_region is not None:
                from .region import region_masks
                parser, classes, r, sigma = edit_region
                mask = region_masks(parser, origin, classes, r, sigma).to(eng.device)
                blend = (mask, ref)
                os.makedirs(folder_dir, exist_ok=True)
                tvu.save_image(tvu.make_grid(mask[:, None].cpu(), nrow=a.bs_train, padding=1),
                               os.path.join(folder_dir, f'{file_name}_ngen{a.n_train_step}_region_mask.png'))
            if region_compose is not None:
                from . import region
                parser, classes, r, sigma, times, row_coeffs = region_compose
                masks = region.compose_masks(parser, origin, classes, r, sigma).to(eng.device)
                os.makedirs(folder_dir, exist_ok=True)
                tvu.save_image(tvu.make_grid(masks.reshape(-1, 1, *masks.shape[2:]).cpu(), nrow=a.bs_train, padding=1),
                               os.path.join(folder_dir, f'{file_name}_ngen{a.n_train_step}_region_compose.png'))
        coeffs = hs_coeff if isinstance(hs_coeff, list) else [hs_coeff]
        edited = []
        if region_compose is not None:
            edited = [self.compose_batch(model, x_lat_tensor, seq_inv, seq_inv_next, masks, ref, times, row_coeffs,
                                         **kw_a)]
        elif sweep_times is not None:
            tpc, chunks = plan_sweep(len(coeffs), bs, getattr(a, "max_rows_per_replay", 16))
            for chunk in chunks:
                rows = sweep_rows(chunk, tpc, bs)
                sch = self.sweep_schedule(seq_inv, seq_inv_next, [sweep_times[k] for k in rows],
                                          [coeffs[k] for k in rows])
                x0 = self.edit_batch(model, pad_rows(x_lat_tensor.repeat(len(chunk), 1, 1, 1), tpc * bs), sch, **kw_a)
                edited += [x0[j * bs:(j + 1) * bs].clone() for j in range(len(chunk))]
        elif not getattr(a, "pass_editing", False):
            # the reference replays the trajectory once per tuple (:495-532); the tuples share x_T and the schedule, so
            # they run as rows of one batch (tuples x images), each row with its own hs_coeff, in chunks of whole tuples
            # of at most --max_rows_per_replay rows.  A sample's result does not depend on its batch neighbours, so
            # every row equals the per-tuple replay bit for bit.
            sch = self.make_schedule(seq_inv, seq_inv_next, coeffs[0])
            edit_ts = [st.t for st in sch.steps if st.edit and st.kind == "ddim"]  # the same for every tuple
            explicit = (not get_delta_hs) and delta_h_dict is not None and any(
                torch.is_tensor(v) for v in delta_h_dict.values())
            kw = {}
            if explicit:  # :517: dict[0] with --ignore_timesteps --train_delta_h, else dict[t] for t >= t_edit
                glob = bool(getattr(a, "ignore_timesteps", False) and getattr(a, "train_delta_h", False))
                rows = []
                for t in edit_ts:
                    dh = delta_h_dict[0] if glob else delta_h_dict[int(t)]
                    if dh is None:
                        raise KeyError(f"no Δh for edit timestep {t} in the checkpoint")
                    dh = dh.detach().float()
                    rows.append(dh[0] if dh.dim() == 4 and dh.shape[0] == 1 else dh)
                if rows:
                    kw["delta_hs"] = torch.stack(rows)
            elif get_delta_hs:
                kw["record_dh"] = True
            if h_direction is not None:
                from .hspace import direction_rows
                dirs = direction_rows(h_direction, edit_ts)
                if dirs is not None:
                    kw["h_direction"] = dirs
            if blend is not None:  # rows are tuple-major blocks of the bs images: row n blends with image n % bs
                kw["blend"] = blend
            kw.update(kw_a)  # anchored rows, like the blend, take image n % bs
            max_rows = getattr(a, "max_rows_per_replay", 16)
            if "delta_hs" in kw and len({float(tup[0]) for tup in coeffs}) > 1:
                max_rows = 0  # explicit Δh takes one slerp weight 1 - c0 per replay: one tuple per chunk
            tpc, chunks = plan_sweep(len(coeffs), bs, max_rows)
            n = eng.n_delta
            # explicit Δh reads only c0, which the chunk's schedule carries; DeltaBlocks read one tuple per row
            per_row = "delta_hs" not in kw and n > 0 and all(len(tup) >= n + 1 for tup in coeffs)
            if "delta_hs" in kw and kw["delta_hs"].dim() == 5:  # per-image Δh rows: repeat them for every tuple row
                kw["delta_hs"] = kw["delta_hs"].repeat(1, tpc, 1, 1, 1)
            for chunk in chunks:
                sch = self.make_schedule(seq_inv, seq_inv_next, coeffs[chunk[0]])
                rows_x = pad_rows(x_lat_tensor.repeat(len(chunk), 1, 1, 1), tpc * bs)
                noise = None
                if sch.n_stochastic and anchors is None:  # the per-tuple draws of the sequential loop, in tuple order
                    noise = chunk_noise(len(chunk), tpc, bs, lambda: torch.randn(
                        (sch.n_stochastic, *x_lat_tensor.shape), device=eng.device))
                if per_row:
                    table = torch.tensor([[float(c) for c in coeffs[i][:n + 1]] for i in chunk for _ in range(bs)],
                                         dtype=torch.float32)
                    kw["hs_coeffs"] = pad_rows(table, tpc * bs)
                elif "h_direction" in kw:  # (c0, α) per row
                    table = torch.tensor([[float(coeffs[i][0]), float(coeffs[i][1])] for i in chunk for _ in range(bs)],
                                         dtype=torch.float32)
                    kw["hs_coeffs"] = pad_rows(table, tpc * bs)
                x0 = self.edit_batch(model, rows_x, sch, noise=noise, record_process=save_process_delta_h, **kw)
                edited += [x0[j * bs:(j + 1) * bs].clone() for j in range(len(chunk))]
                if save_process_delta_h and chunk is chunks[-1]:  # each tuple rewrote these files: the last one stays
                    j = len(chunk) - 1
                    self._write_process(eng, sch, os.path.join(folder_dir, file_name), "delta_h", bs,
                                        rows=slice(j * bs, (j + 1) * bs))
                if get_delta_hs:  # accumulated tuple by tuple, as the per-tuple loop adds them
                    rec = eng.last_records["delta_h"].cpu()
                    for j in range(len(chunk)):
                        for ei, t in enumerate(edit_ts):
                            r = rec[ei][j * bs:(j + 1) * bs]
                            delta_h_dict[int(t)] = r if delta_h_dict.get(int(t)) is None else delta_h_dict[int(t)] + r
        x_list += edited
        os.makedirs(folder_dir, exist_ok=True)
        tvu.save_image(tvu.make_grid((torch.cat(x_list, dim=0) + 1) * 0.5, nrow=a.bs_train, padding=1),
                       os.path.join(folder_dir, f'{file_name}_ngen{a.n_train_step}.png'))
        if scorers is not None:
            scorers.score(file_name, folder_dir, mode, batch_ids, origin, edited, coeffs, x0_source)
        print(f'{time.time() - time_s} seconds, {file_name}_ngen{a.n_train_step}.png is saved')
        return x_list

    # ------------------------------------------------------------------------------------------
    def load_lpips(self):
        """LPIPS-Alex from --lpips_weights (a torch.save of the lpips package's LPIPS(net='alex').state_dict()), or
        seeded synthetic weights with --synthetic_weights, as load_pretrained_model does for the UNet"""
        from .lpips import LPIPS
        a = self.args
        path = getattr(a, "lpips_weights", None)
        if path:
            return LPIPS(path, device=self.device)
        if getattr(a, "synthetic_weights", False):
            from .synthetic import lpips_state_dict
            return LPIPS(lpips_state_dict(seed=getattr(a, "seed", 1234)), device=self.device)
        raise FileNotFoundError("no --lpips_weights given: the LPIPS-Alex weights cannot be downloaded here (pass "
                                "--lpips_weights <state dict of lpips.LPIPS(net='alex')> or --synthetic_weights)")

    @torch.no_grad()
    def lpips_batch(self, model, loss_fn, x0, seq_inv, seq_inv_next, image_folder=None):
        """One inversion replay of the images x0 [B,3,S,S] with the LPIPS launches in the graph
        (compute_lpips_distance's per-image loop, diffusion_latent.py:1244-1273).  Returns, per image, the lists
        (LPIPS(x_t, x0) per step, LPIPS(x0_t, x0) per step) over the steps zip(seq_inv_next[1:], seq_inv[1:]).
        image_folder: also write x_t and x0_t of every step of row 0 as LPIPS_0_{t_next}.png / X0_t_LPIPS_0_{t_next}.png"""
        import torchvision.utils as tvu
        eng = model.engine
        sch = Schedule.inversion(self.betas, seq_inv, seq_inv_next)
        eng.sample(x0.to(eng.device), sch, lpips=loss_fn, record_process=image_folder is not None)
        rec = eng.last_records
        if image_folder is not None:
            for k, st in enumerate(sch.steps):
                tvu.save_image((rec["x"][k][:1] + 1) * 0.5, os.path.join(image_folder, f"LPIPS_0_{st.t_next}.png"))
                tvu.save_image((rec["x0_t"][k][:1] + 1) * 0.5,
                               os.path.join(image_folder, f"X0_t_LPIPS_0_{st.t_next}.png"))
        lx, lx0 = rec["lpips_x"].cpu(), rec["lpips_x0_t"].cpu()  # [steps][B]
        return [(lx[:, i].tolist(), lx0[:, i].tolist()) for i in range(x0.shape[0])]

    @torch.no_grad()
    def compute_lpips_distance(self):
        """--lpips (diffusion_latent.py:1191-1303): invert the first n_train_img + 1 images of
        --custom_train_dataset_dir with n_inv_step DDIM steps, take LPIPS-Alex of x_t and of x0_t against the image after
        every step, and write the per-t mean and std (np.mean / np.std over the images) as
        <config stem>_LPIPS_distance_{x,x_std,x0_t,x0_t_std}.tsv into --lpips_table_dir (default utils), where
        set_t_edit_t_addnoise reads them.  The first image runs alone and leaves its per-step PNGs in image_folder;
        the others run bs_train per replay (every row's distances equal its batch-1 run bit for bit)."""
        import torchvision.utils as tvu
        a = self.args
        self.edit_region_setup()  # refuses --lpips
        self.region_compose_setup()  # refuses --lpips
        self.exact_inversion_setup()  # refuses --lpips
        if getattr(a, "content_preservation", False):
            self.content_preservation_setup()  # refuses --lpips
        if getattr(a, "dino_structure", False):
            self.dino_structure_setup()  # refuses --lpips
        if self.world > 1:
            raise NotImplementedError("--lpips computes statistics over every image: run single-process")
        print("Get lpips distance...")
        seq_inv = [int(s + 1e-6) for s in list(np.linspace(0, 1, a.n_inv_step) * a.t_0)]
        seq_inv_next = [-1] + list(seq_inv[:-1])
        folder = getattr(a, "custom_train_dataset_dir", None)
        if not folder or not os.path.isdir(folder):
            raise FileNotFoundError(f"--custom_train_dataset_dir {folder!r} is not a directory: no images to invert")
        # the reference's loader loop breaks after processing step n_train_img: n_train_img + 1 images
        imgs = _load_image_folder(folder, self.config.data.image_size, a.n_train_img + 1)
        if not imgs:
            raise FileNotFoundError(f"no png/jpg images in {folder}")
        model = self.load_pretrained_model().to(self.device)
        loss_fn = self.load_lpips()
        image_folder = getattr(a, "image_folder", None) or os.path.join(a.exp, "image_samples")
        os.makedirs(image_folder, exist_ok=True)
        tvu.save_image((imgs[0] + 1) * 0.5, os.path.join(image_folder, "LPIPS_0_0_orig.png"))
        per_image = self.lpips_batch(model, loss_fn, imgs[0], seq_inv, seq_inv_next, image_folder=image_folder)
        rest = imgs[1:]
        bs = min(max(1, a.bs_train), max(1, len(rest)))
        for k in range(0, len(rest), bs):  # every replay bs rows (the last one padded): one captured graph
            chunk = rest[k:k + bs]
            per_image += self.lpips_batch(model, loss_fn, pad_rows(torch.cat(chunk), bs), seq_inv,
                                          seq_inv_next)[:len(chunk)]
        tables = lpips_tables(seq_inv, seq_inv_next, per_image)
        tdir = getattr(a, "lpips_table_dir", None) or "utils"
        os.makedirs(tdir, exist_ok=True)
        stem = os.path.basename(str(a.config).split(".")[0])
        for suffix, text in tables.items():
            with open(os.path.join(tdir, f"{stem}_LPIPS_distance_{suffix}.tsv"), "w") as f:
                f.write(text)
        return tables

    # ------------------------------------------------------------------------------------------
    def checkpoint_name(self):
        """the Δh checkpoint run_test loads (:594-614); --multiple_attr and --attr_sweep replace 'attribute' in it"""
        a = self.args
        exp_id = os.path.split(a.exp)[-1]
        ckdir = getattr(a, "checkpoint_dir", "checkpoint")
        if a.load_from_checkpoint:
            save_name = (f'{ckdir}/{a.load_from_checkpoint}_LC_{self.config.data.category}_t{a.t_0}_ninv'
                         f'{a.n_inv_step}_ngen{a.n_train_step}_{a.n_iter - 1}.pth')
        else:
            save_name = f'{ckdir}/{exp_id}_{a.n_iter - 1}.pth'
        if a.manual_checkpoint_name:
            save_name = os.path.join(ckdir, a.manual_checkpoint_name)
        elif a.choose_checkpoint_num:
            save_name = save_name[:-4] + f'_{a.choose_checkpoint_num}.pth'
        return save_name

    def _batches(self, pairs, keep_source):
        """this rank's batches of the latents of run_test and run_attr_sweep (:779-874): (mode, step, x_T, x0, image
        indices, x0_source) per batch of the [x0, x_rec, x_T] triples of pairs[mode], step the last image's index.
        Images before --start_image_id or outside --target_image_id are left out but count towards the batch boundary
        (step + 1) % bs_train; the batches go round-robin to the ranks, every batch counted; a pass ends at its last
        image (n_train_img / n_test_img).  x0 with --use_x0_tensor, x0_source (the images the latents were inverted
        from) with keep_source, else None."""
        a = self.args
        target_ids = [int(i) for i in str(a.target_image_id).split(" ")] if getattr(a, "target_image_id", None) \
            else None
        for mode, do, n_img in (("train", a.do_train, a.n_train_img), ("test", a.do_test, a.n_test_img)):
            if not do:
                continue
            batch, batch_idx = [], 0
            for step, (x0, _, x_lat) in enumerate(pairs[mode]):
                if (target_ids is not None and step not in target_ids) or a.start_image_id > step:
                    continue
                batch.append((step, x0, x_lat))
                if (step + 1) % a.bs_train != 0:
                    continue
                if batch_idx % self.world == self.rank:  # batch-sharded across ranks, no per-step communication
                    x0s = torch.cat([x for _, x, _ in batch])
                    yield (mode, step, torch.cat([x for _, _, x in batch]), x0s if a.use_x0_tensor else None,
                           [i for i, _, _ in batch], x0s if keep_source else None)
                batch_idx += 1
                if step == n_img - 1:
                    break
                batch = []

    @torch.no_grad()
    def anchor_batch(self, model, x0):
        """--exact_inversion: the inversion.Anchors of the input images x0 [B][C][S][S] (UNetEngine.anchors on the
        --n_inv_step DDIM inversion grid), on the device"""
        a = self.args
        seq, seq_next = make_sequences(a.t_0, a.n_inv_step)
        eng = model.engine
        return eng.anchors(x0.to(eng.device), Schedule.inversion(self.betas, seq, seq_next))

    def _edit_batches(self, model, pairs, scorers, exact):
        """_batches, with the batch's anchors appended (None without --exact_inversion).  Anchored, x_T is the
        anchors' A[0], inverted here from the batch's input images; the cached x_T of the pairs is not used."""
        for mode, step, x_lat, x0, ids, x0_source in self._batches(pairs, scorers.keeps_source or exact):
            anchors = None
            if exact:
                anchors = self.anchor_batch(model, x0_source)
                x_lat = anchors.x_T
                x0_source = x0_source if scorers.keeps_source else None
            yield mode, step, x_lat, x0, ids, x0_source, anchors

    @torch.no_grad()
    def run_test(self):
        a = self.args
        exact = self.exact_inversion_setup()
        scoring.fid_options_check(self)
        compose_spec = self.region_compose_setup()  # refuses --attr_sweep, --edit_region and --h_direction too
        region_spec = self.edit_region_setup()  # refuses --attr_sweep too, before it is dispatched
        h_dir_path = self.h_direction_setup()  # refuses --attr_sweep too, before it is dispatched
        if compose_spec is not None:
            return self.run_region_compose(compose_spec)
        if getattr(a, "attr_sweep", ""):
            return self.run_attr_sweep()
        print("Running Test")
        if getattr(a, "warigari", 0.0):
            print("--warigari is accepted and has no effect (the reference's branch returns the same values, "
                  "utils/diffusion_utils.py:103-109)")
        scorers = scoring.Scorers(self)
        if a.multiple_attr and self.needs_clip() and self.clip_configured():
            cosine = self.choose_attribute(a.multiple_attr.split(' '))  # :640-652
            self.set_t_edit_t_addnoise(LPIPS_th=a.lpips_edit_th, LPIPS_addnoise_th=a.lpips_addnoise_th, cosine=cosine)
        else:
            self.set_t_edit_t_addnoise(LPIPS_th=a.lpips_edit_th, LPIPS_addnoise_th=a.lpips_addnoise_th)
        # ----------- sequences (:560-574)
        if a.n_train_step != 0:
            seq_train = np.linspace(0, 1, a.n_train_step) * a.t_0
            seq_train = [int(s + 1e-6) for s in list(seq_train[seq_train >= self.t_edit])]
        else:
            seq_train = list(range(self.t_edit, a.t_0))
        seq_test_f = np.linspace(0, 1, a.n_test_step) * a.t_0
        seq_test_edit = [int(s + 1e-6) for s in list(seq_test_f[seq_test_f >= self.t_edit])]
        seq_test = [int(s + 1e-6) for s in list(seq_test_f)]
        seq_test_next = [-1] + list(seq_test[:-1])
        # ----------- model
        model = self.load_pretrained_model()
        delta_h_dict = {i: None for i in seq_train}
        if a.train_delta_block:
            model.setattr_layers(a.get_h_num)
        # ----------- Δh checkpoint name resolution (:594-614)
        exp_id = os.path.split(a.exp)[-1]
        save_name = self.checkpoint_name()
        # ----------- global / mean Δh (:616-627): load the cached dict if it exists, else compute it below
        num_mean, load_dict = a.num_mean_of_delta_hs, False
        train_delta_h, train_delta_block = bool(getattr(a, "train_delta_h", False)), bool(a.train_delta_block)
        latent_name = f"checkpoint_latent/{exp_id}_{a.n_test_step}_{num_mean}.pth"
        if num_mean:
            if self.world > 1:
                raise NotImplementedError("--num_mean_of_delta_hs accumulates over consecutive images: run single-process")
            if os.path.isfile(latent_name):
                save_name, load_dict = latent_name, True
                delta_h_dict = {i: None for i in seq_test}
        scaling_factor = a.n_train_step / a.n_test_step * a.hs_coeff_delta_h  # :626
        h_direction = None
        if h_dir_path is not None:
            from .hspace import load_direction
            h_direction = load_direction(h_dir_path, self.config, a, model.arch.mid_ch)
            hs_coeff = h_direction_coeffs(a)
        elif a.multiple_attr:
            attrs = a.multiple_attr.split(' ')
            coeffs = [float(c) for c in a.multiple_hs_coeff.split(' ')] if a.multiple_hs_coeff else []
            coeffs = coeffs + [1.0] * (len(attrs) - len(coeffs))
            save_name_list = [save_name.replace('attribute', attr) for attr in attrs]
            hs_coeff = tuple([1.0 * a.hs_coeff_origin_h] +
                             [1.0 / (len(attrs)) ** 0.5 * scaling_factor * c for c in coeffs])  # :654
        else:
            save_name_list = [save_name]
            hs_coeff = (1.0 * a.hs_coeff_origin_h, 1.0 * scaling_factor)  # :659
        # ----------- load (:662-697)
        if h_direction is not None:
            pass  # the direction replaces the Δh checkpoint
        elif os.path.exists(save_name_list[0]):
            print(f'{save_name} exists. load checkpoint')
            if train_delta_block:
                if num_mean and load_dict:  # the cached mean Δh replaces the DeltaBlock (:669-672)
                    train_delta_h, train_delta_block, num_mean = True, False, 0
                else:
                    for i in range(a.get_h_num):
                        ck = torch.load(save_name_list[i], map_location="cpu", weights_only=True)
                        getattr(model, f"layer_{i}").load_state_dict(ck["0"])  # :674-676
            if train_delta_h:
                saved = torch.load(save_name_list[0], map_location="cpu", weights_only=True)

                def get(k):  # string keys (run_training's torch.save) or int keys (the mean-Δh cache); a timestep
                    return saved[f"{k}"] if f"{k}" in saved else saved.get(k)  # below t_edit has no entry

                if getattr(a, "ignore_timesteps", False):  # global Δh is delta_h_dict[0]
                    delta_h_dict[0] = get(0)
                else:
                    for i in list(delta_h_dict.keys()):
                        delta_h_dict[i] = get(i)
        elif num_mean:
            print("There in no pre-computed mean of delta_hs! Now compute it...")
        else:
            raise FileNotFoundError(f"checkpoint({save_name_list[0]}) does not exist!")
        # ----------- train-step keys -> test-step keys (:699-724)
        if a.n_train_step != a.n_test_step:
            if train_delta_h:
                if not load_dict:
                    test_dict, trained_idx = {}, 0
                    if getattr(a, "ignore_timesteps", False):
                        test_dict[0] = delta_h_dict[0]
                    interval = (seq_train[1] - seq_train[0]) if len(seq_train) > 1 else 0
                    for i in seq_test_edit:
                        test_dict[i] = delta_h_dict[seq_train[trained_idx]]
                        if i > seq_train[trained_idx] - interval and trained_idx < len(seq_train) - 1:
                            trained_idx += 1
                    delta_h_dict = test_dict
            else:
                for i in seq_test:
                    delta_h_dict.setdefault(i, None)
        a_train_delta_h_prev = getattr(a, "train_delta_h", False)
        a.train_delta_h = train_delta_h  # save_image's global-Δh rule reads it (:517)
        if a.delta_interpolation and h_direction is None:  # :726-755
            vals = np.linspace(a.min_delta, a.max_delta, a.num_delta).tolist()
            if a.multiple_attr:
                assert a.get_h_num == 2, "delta_multiple_attr_interpolation is only supported for get_h_num == 2"
                hs_coeff = [(1.0, v1 * hs_coeff[1], v2 * hs_coeff[2]) for v1 in vals for v2 in vals]
            else:
                hs_coeff = [tuple([1.0] + [v * e for e in hs_coeff[1:]]) for v in vals]
        if num_mean:
            assert a.bs_train == 1, "if you want to use mean, batch_size must be 1"
        model = model.to(self.device)
        if self.world > 1 and torch.distributed.is_initialized():
            broadcast_weights(model)
        # ----------- x_T
        if a.load_random_noise:
            pairs = self.random_noise_pairs(model, saved_noise=bool(getattr(a, "saved_random_noise", False)))
        else:
            pairs = self.precompute_pairs(model)
        if getattr(a, "target_image_id", None):
            assert a.bs_train == 1, "target_image_id is only supported for batch_size == 1"
        results = {}
        try:
            with scorers:
                edit_region = None
                if region_spec is not None:  # --seg_consistency's parser serves the masks too
                    from .face_parsing import FaceParser
                    classes, r, sigma, seg_sd = region_spec
                    region_spec = None
                    edit_region = (scorers.nets.get("seg") or FaceParser(seg_sd, device=self.device), classes, r, sigma)
                for mode, step, x_lat, x0, ids, x0_source, anchors in self._edit_batches(model, pairs, scorers, exact):
                    results[(mode, step)] = self.save_image(
                        model, x_lat, seq_test, seq_test_next, save_x0=a.save_x0, save_x_origin=a.save_x_origin,
                        x0_tensor=x0, delta_h_dict=delta_h_dict, get_delta_hs=bool(num_mean),
                        save_process_origin=bool(getattr(a, "save_process_origin", False)),
                        save_process_delta_h=bool(getattr(a, "save_process_delta_h", False)),
                        folder_dir=a.test_image_folder, file_name=f'{mode}_{step}_{a.n_iter - 1}', hs_coeff=hs_coeff,
                        h_direction=h_direction, scorers=scorers, mode=mode, batch_ids=ids, x0_source=x0_source,
                        edit_region=edit_region, **({"anchors": anchors} if exact else {}))
                    # the last image of the pass ends it before the mean is taken
                    if mode == "train" and num_mean and step == num_mean - 1 and step != a.n_train_img - 1:
                        # mean over the first num_mean images per timestep, key 0 = mean over timesteps (:811-832)
                        for k in delta_h_dict:
                            if delta_h_dict[k] is not None:
                                delta_h_dict[k] = delta_h_dict[k] / (step + 1)
                        tot, cnt = None, 0
                        for k in list(delta_h_dict.keys()):
                            if delta_h_dict[k] is None:
                                continue
                            tot = delta_h_dict[k].clone() if tot is None else tot + delta_h_dict[k]
                            cnt += 1
                        delta_h_dict[0] = tot / cnt
                        os.makedirs("checkpoint_latent", exist_ok=True)
                        _atomic_save(delta_h_dict, latent_name)
                        print(f'Dict: {latent_name} is saved.')
                        num_mean = 0
                        print("now we use mean of delta_hs")
                scorers.finish(hs_coeff if isinstance(hs_coeff, list) else [hs_coeff])
                edit_region = None  # the parser goes with the scorers' networks, and the CUDA cache after it
        finally:
            a.train_delta_h = a_train_delta_h_prev
        self.last_delta_h_dict = delta_h_dict
        return results


    # ------------------------------------------------------------------------------------------
    def exact_inversion_setup(self):
        """--exact_inversion's requirements, checked before any model loads: False without the flag, else True.
        ValueError with the reason."""
        a = self.args
        if not getattr(a, "exact_inversion", False):
            return False
        if not getattr(a, "run_test", False):
            raise ValueError("--exact_inversion anchors the edits of --run_test to their input images: add --run_test")
        for flag, on, why in (
                ("--load_random_noise", getattr(a, "load_random_noise", False), "a random latent has no input image"),
                ("--saved_random_noise", getattr(a, "saved_random_noise", False), "a random latent has no input image"),
                ("--sample_type ddpm", getattr(a, "sample_type", "ddim") == "ddpm",
                 "the ancestral step has no anchored form"),
                ("--origin_process_addnoise", getattr(a, "origin_process_addnoise", False),
                 "there is no origin pass: the origin is the input image"),
                ("--save_process_origin", getattr(a, "save_process_origin", False),
                 "there is no origin pass: the origin is the input image"),
                ("--lpips", getattr(a, "lpips", False), "it edits nothing"),
                ("--diff_style", getattr(a, "diff_style", False), "it is not a --run_test edit"),
                ("--h_directions", getattr(a, "h_directions", False), "it edits nothing"),
                ("--num_mean_of_delta_hs", getattr(a, "num_mean_of_delta_hs", 0),
                 "the mean Δh must come from the unanchored pass")):
            if on:
                raise ValueError(f"--exact_inversion does not combine with {flag}: {why}")
        if a.n_test_step != a.n_inv_step:
            raise ValueError(f"--exact_inversion needs --n_test_step equal to --n_inv_step: the edit steps run on the "
                             f"inversion's grid, got {a.n_test_step} and {a.n_inv_step}")
        return True

    def edit_region_setup(self):
        """--edit_region's requirements, checked before any model loads: None without the flag, else (class indices,
        --edit_region_dilate, --edit_region_feather, the --seg_weights state dict).  ValueError with the reason."""
        from . import region
        a = self.args
        text = getattr(a, "edit_region", None)
        if not text:
            return None
        if not getattr(a, "run_test", False):
            raise ValueError("--edit_region restricts the edits of --run_test: add --run_test")
        for flag, on, why in (
                ("--attr_sweep", getattr(a, "attr_sweep", ""), "its rows follow per-row schedules"),
                ("--diff_style", getattr(a, "diff_style", False), "it is not a --run_test edit"),
                ("--lpips", getattr(a, "lpips", False), "it edits nothing"),
                ("--h_directions", getattr(a, "h_directions", False), "it edits nothing"),
                ("--pass_editing", getattr(a, "pass_editing", False), "nothing is edited"),
                ("--num_mean_of_delta_hs", getattr(a, "num_mean_of_delta_hs", 0),
                 "the mean Δh must come from the unmasked pass")):
            if on:
                raise ValueError(f"--edit_region does not combine with {flag}: {why}")
        classes = region.parse_classes(text)
        r, sigma = getattr(a, "edit_region_dilate", 0), getattr(a, "edit_region_feather", 0.0)
        region.check_options(r, sigma, self.config.data.image_size)
        return classes, r, float(sigma), scoring.seg_weights(self, "--edit_region")

    def region_compose_setup(self):
        """--region_compose's requirements, checked before any model loads: None without the flag, else (attributes,
        the class indices of each, --edit_region_dilate, --edit_region_feather, the --seg_weights state dict, the
        attributes' DeltaBlock checkpoints).  ValueError with the reason."""
        from . import region
        a = self.args
        text = getattr(a, "region_compose", None)
        if not text:
            return None
        if not getattr(a, "run_test", False):
            raise ValueError("--region_compose composes the edits of --run_test: add --run_test")
        each = "every attribute edits with its own DeltaBlock"
        for flag, on, why in (
                ("--attr_sweep", getattr(a, "attr_sweep", ""), "it gives every attribute an image of its own"),
                ("--edit_region", getattr(a, "edit_region", None), "every attribute takes its region from "
                                                                  "--region_compose"),
                ("--multiple_attr", getattr(a, "multiple_attr", ""), each),
                ("--delta_interpolation", getattr(a, "delta_interpolation", False), "a composite has one strength"),
                ("--num_mean_of_delta_hs", getattr(a, "num_mean_of_delta_hs", 0), each),
                ("--train_delta_h", getattr(a, "train_delta_h", False), each),
                ("--h_direction", getattr(a, "h_direction", None), each),
                ("--pass_editing", getattr(a, "pass_editing", False), "nothing is edited"),
                ("--diff_style", getattr(a, "diff_style", False), "it is not a --run_test edit"),
                ("--lpips", getattr(a, "lpips", False), "it edits nothing"),
                ("--h_directions", getattr(a, "h_directions", False), "it edits nothing"),
                ("--DirectionalClipSmilarity", getattr(a, "DirectionalClipSmilarity", False),
                 "a composite has no single source / target text pair"),
                ("--save_process_delta_h", getattr(a, "save_process_delta_h", False),
                 "the rows of a composite are not one edit's trajectory")):
            if on:
                raise ValueError(f"--region_compose does not combine with {flag}: {why}")
        spec = region.parse_compose(text)
        attrs = [attr for attr, _ in spec]
        max_rows = getattr(a, "max_rows_per_replay", 16)
        if len(attrs) > max_rows:
            raise ValueError(f"--region_compose: {len(attrs)} attributes need {len(attrs)} rows per image, above "
                             f"--max_rows_per_replay {max_rows}")
        paths = self.attribute_blocks_setup("--region_compose", attrs)
        r, sigma = getattr(a, "edit_region_dilate", 0), getattr(a, "edit_region_feather", 0.0)
        region.check_options(r, sigma, self.config.data.image_size)
        return (attrs, [classes for _, classes in spec], r, float(sigma), scoring.seg_weights(self, "--region_compose"),
                paths)

    def h_direction_setup(self):
        """--h_direction's requirements, checked before any model loads: the path (None without the flag); ValueError
        when it is combined with a flag that selects another source of Δh"""
        a = self.args
        path = getattr(a, "h_direction", None)
        if not path:
            return None
        for flag, on in (("--train_delta_block", bool(getattr(a, "train_delta_block", False))),
                         ("--train_delta_h", bool(getattr(a, "train_delta_h", False))),
                         ("--multiple_attr", bool(getattr(a, "multiple_attr", ""))),
                         ("--num_mean_of_delta_hs", bool(getattr(a, "num_mean_of_delta_hs", 0))),
                         ("--attr_sweep", bool(getattr(a, "attr_sweep", "")))):
            if on:
                raise ValueError(f"--h_direction replaces the Δh checkpoint: it does not combine with {flag}")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"--h_direction {path!r} is not a file")
        return path

    def h_directions_setup(self):
        """--h_directions' requirements, checked before any model loads: ('pca', K) or ('mean_diff', (pos, neg))"""
        a = self.args
        K = getattr(a, "h_pca", None)
        pos, neg = getattr(a, "h_pos_dir", None), getattr(a, "h_neg_dir", None)
        if (K is not None) == bool(pos or neg):
            raise ValueError("--h_directions needs exactly one mode: --h_pca K, or --h_pos_dir A --h_neg_dir B")
        if self.world > 1:
            raise ValueError("--h_directions computes statistics over every sample: run it single-process, not under "
                             "torchrun")
        if not getattr(a, "h_direction_out", None):
            raise ValueError("--h_directions needs --h_direction_out DIR for the direction files")
        if K is not None:
            if K < 1 or K > a.n_train_img - 1:
                raise ValueError(f"--h_pca {K}: between 1 and n_train_img - 1 = {a.n_train_img - 1} components "
                                 "(n samples have at most n - 1 principal directions)")
            return "pca", K
        if not (pos and neg):
            raise ValueError("--h_pos_dir and --h_neg_dir go together")
        for flag, d in (("h_pos_dir", pos), ("h_neg_dir", neg)):
            if not os.path.isdir(d) or not image_paths(d):
                raise ValueError(f"--{flag} {d!r} is not a directory holding png / jpg images")
        return "mean_diff", (pos, neg)

    @torch.no_grad()
    def run_h_directions(self, keep_h=False):
        """--h_directions: the plain generative pass (run_test's origin pass) over the n_test_step grid from every
        latent, with h recorded at every step, bs_train rows per replay; then per step the PCA of h over the latents
        or the mean difference of two sets.  Writes hspace.py's direction files and h_directions.tsv into
        --h_direction_out; returns their paths.
          --h_pca K: the n_train_img "train" latents run_test would use: random noise with --load_random_noise, else
            the --custom_train_dataset_dir images inverted by precompute_pairs (its cache is shared with run_test).
          --h_pos_dir A --h_neg_dir B: the first n_train_img images of each folder (sorted by name), DDIM-inverted.
        The device memory of the recorded h ([steps][n][d] fp32) is checked before any inversion or generation.
        keep_h: keep that buffer as self.h_directions_x (otherwise it is released when the run ends)."""
        from . import hspace
        a = self.args
        self.edit_region_setup()  # refuses --h_directions
        self.region_compose_setup()  # refuses --h_directions
        self.exact_inversion_setup()  # refuses --h_directions
        if getattr(self.args, "dino_structure", False):
            self.dino_structure_setup()  # refuses --h_directions
        mode, arg = self.h_directions_setup()
        seq, seq_next = make_sequences(a.t_0, a.n_test_step)
        size = self.config.data.image_size
        bs = max(1, a.bs_train)
        if mode == "pca":
            folder = None if a.load_random_noise else getattr(a, "custom_train_dataset_dir", None)
            if not a.load_random_noise and (not folder or not os.path.isdir(folder)):
                raise FileNotFoundError(f"--custom_train_dataset_dir {folder!r} is not a directory: nothing to invert "
                                        "(use --load_random_noise for random latents)")
            n = a.n_train_img if folder is None else min(a.n_train_img, len(image_paths(folder)))
            if n < arg + 1:
                raise ValueError(f"--h_pca {arg} needs {arg + 1} latents; {folder!r} holds {n} images")
        else:
            n_pos, n_neg = (min(a.n_train_img, len(image_paths(f))) for f in arg)
            n = n_pos + n_neg
        sch = self.make_schedule(seq, seq_next, (1.0,), edit=False, addnoise=False)
        model = self.load_pretrained_model().to(self.device)
        eng = model.engine
        shape = tuple(eng.plan(bs).mid_f32.shape[1:])
        d, steps = int(np.prod(shape)), len(sch.steps)
        need = steps * n * d * 4
        free, _ = torch.cuda.mem_get_info(eng.device)
        if need > free:
            raise MemoryError(f"--h_directions: h of {steps} steps x {n} samples x {d} features takes "
                              f"{need / 2**30:.2f} GiB; the device has {free / 2**30:.2f} GiB free (lower --n_train_img)")
        if mode == "pca":
            pairs = (self.random_noise_pairs(model) if a.load_random_noise else
                     self.precompute_pairs(model, modes=("train",)))["train"]
            x_T = torch.cat([p[2] for p in pairs[:n]])
            n_pos = None
        else:
            def invert(folder):  # only x_T is needed: no reconstruction pass
                imgs = _load_image_folder(folder, size, a.n_train_img)
                return torch.cat([self.invert_batch(model, torch.cat(imgs[k:k + bs]), reconstruct=False)[0]
                                  for k in range(0, len(imgs), bs)])
            x_T = torch.cat([invert(arg[0]), invert(arg[1])])
        if x_T.shape[0] != n:  # a pairs cache written from another state of the folder
            raise ValueError(f"--h_directions: {x_T.shape[0]} latents for {n} images; rerun with --re_precompute")
        X = torch.empty((steps, n, d), dtype=torch.float32, device=eng.device)
        for k in range(0, n, bs):  # every replay bs rows (the last one padded): one captured graph
            m = min(bs, n - k)
            self.edit_batch(model, pad_rows(x_T[k:k + m], bs), sch, record_h=True)
            X[:, k:k + m].copy_(eng.last_records["h"][:, :m].reshape(steps, m, d))
        directions, rows = hspace.discover(X, [st.t for st in sch.steps], K=arg if mode == "pca" else None,
                                           n_pos=n_pos)
        meta = {"category": self.config.data.category, "mid_ch": int(model.arch.mid_ch), "t_0": int(a.t_0),
                "n_test_step": int(a.n_test_step), "n": n if mode == "pca" else {"pos": n_pos, "neg": n - n_pos}}
        self.h_directions = directions
        if keep_h:
            self.h_directions_x = X
        del X
        paths = hspace.write_directions(a.h_direction_out, directions, rows, shape, meta)
        for p in paths:
            print(f"{p} is saved")
        return paths

    # ------------------------------------------------------------------------------------------
    def attr_sweep_setup(self):
        """--attr_sweep's requirements, checked before any model is loaded; raises ValueError with the reason.
        Returns (attributes, their DeltaBlock checkpoints): the checkpoint name with 'attribute' replaced by each
        attribute, as --multiple_attr resolves them."""
        a = self.args
        attrs = [t for t in str(a.attr_sweep).split(" ") if t]
        if not attrs:
            raise ValueError("--attr_sweep names no attribute")
        if len(set(attrs)) != len(attrs):
            raise ValueError(f"--attr_sweep names an attribute twice: {attrs}")
        for flag, on in (("--multiple_attr", bool(a.multiple_attr)), ("--delta_interpolation", a.delta_interpolation),
                         ("--num_mean_of_delta_hs", bool(a.num_mean_of_delta_hs)),
                         ("--train_delta_h", bool(getattr(a, "train_delta_h", False)))):
            if on:
                raise ValueError(f"--attr_sweep edits with one DeltaBlock per attribute: it does not combine with {flag}")
        return attrs, self.attribute_blocks_setup("--attr_sweep", attrs)

    def attribute_blocks_setup(self, flag, attrs):
        """the requirements of a mode whose rows edit with one DeltaBlock per attribute (`flag`: --attr_sweep,
        --region_compose): per-row DDIM schedules, one block per checkpoint, every image edited.  Returns the
        checkpoints, the checkpoint name with 'attribute' replaced by each attribute, as --multiple_attr resolves them."""
        a = self.args
        if getattr(a, "sample_type", "ddim") != "ddim":
            raise ValueError(f"{flag} needs --sample_type ddim (every row its own eta schedule), got "
                             f"{a.sample_type!r}")
        if a.get_h_num != 1:
            raise ValueError(f"{flag} loads one DeltaBlock per attribute: --get_h_num must be 1, got {a.get_h_num}")
        if getattr(a, "pass_editing", False):
            raise ValueError(f"{flag} edits every image: it does not combine with --pass_editing")
        name = self.checkpoint_name()
        if "attribute" not in os.path.basename(name):
            raise ValueError(f"{flag}: the checkpoint name {name!r} has no 'attribute' to replace by each "
                             "attribute (e.g. --manual_checkpoint_name attribute_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth)")
        dirname, base = os.path.split(name)
        paths = [os.path.join(dirname, base.replace("attribute", attr)) for attr in attrs]
        missing = [p for p in paths if not os.path.isfile(p)]
        if missing:
            raise ValueError(f"{flag}: checkpoint(s) {missing} do not exist")
        return paths

    def attr_sweep_schedules(self, attrs):
        """(t_edit, t_addnoise) of every attribute: --user_defined_t_edit / --user_defined_t_addnoise for all of them,
        else set_t_edit_t_addnoise with the attribute's CLIP text cosine, the K cosines from one clip_cosines call
        (or --clip_cosine for all)"""
        a = self.args
        cosines = [None] * len(attrs)
        both = getattr(a, "user_defined_t_edit", None) is not None and \
            getattr(a, "user_defined_t_addnoise", None) is not None
        if not both and self.needs_clip() and self.clip_configured():
            cosines = self.clip_cosines([self.edit_texts(attr) for attr in attrs])
        out = []
        for attr, cos in zip(attrs, cosines):
            self.set_t_edit_t_addnoise(LPIPS_th=a.lpips_edit_th, LPIPS_addnoise_th=a.lpips_addnoise_th, cosine=cos)
            out.append((int(self.t_edit), int(self.t_addnoise)))
            print(f"attribute {attr}: t_edit {out[-1][0]}, t_addnoise {out[-1][1]}")
        return out

    @torch.no_grad()
    def run_attr_sweep(self):
        """--run_test --attr_sweep "a b ..": every image edited with every attribute in one batched trajectory per
        chunk of rows (attributes x images).  Row (attribute k, image i) is what --run_test --edit_attr <k> gives
        image i: the attribute's own DeltaBlock, t_edit and t_addnoise (schedule.RowSchedule)."""
        a = self.args
        print("Running Test (attribute sweep)")
        attrs, paths = self.attr_sweep_setup()
        exact = self.exact_inversion_setup()
        scorers = scoring.Scorers(self, attrs)
        times = self.attr_sweep_schedules(attrs)
        self.sweep_times = dict(zip(attrs, times))
        seq_test = [int(s + 1e-6) for s in list(np.linspace(0, 1, a.n_test_step) * a.t_0)]
        seq_test_next = [-1] + list(seq_test[:-1])
        model, coeffs, pairs = self.attribute_run(paths)
        results = {}
        with scorers:
            for mode, step, x_lat, x0, ids, x0_source, anchors in self._edit_batches(model, pairs, scorers, exact):
                results[(mode, step)] = self.save_image(
                    model, x_lat, seq_test, seq_test_next, save_x0=a.save_x0, save_x_origin=a.save_x_origin,
                    x0_tensor=x0, folder_dir=a.test_image_folder, file_name=f'{mode}_{step}_{a.n_iter - 1}',
                    hs_coeff=coeffs, sweep_times=times, scorers=scorers, mode=mode, batch_ids=ids, x0_source=x0_source,
                    **({"anchors": anchors} if exact else {}))
            scorers.finish(coeffs)
        return results

    def attribute_run(self, paths):
        """what a run with one DeltaBlock per attribute (--attr_sweep, --region_compose) edits with: (the model with the
        blocks of `paths` packed as layer_0 .. layer_{K-1} on the device, the coefficients of each attribute's rows,
        the latents)"""
        a = self.args
        K = len(paths)
        model = self.load_pretrained_model()
        # the latents below come from the global random stream, after the model is built: advance it as run_test does
        # (one DeltaBlock's default init), then create the K blocks, whose initial values the checkpoints replace,
        # without touching it, so that every image gets the x_T of its --edit_attr run
        model.setattr_layers(a.get_h_num)
        with torch.random.fork_rng(devices=[]):
            model.setattr_layers(K)
        for i, path in enumerate(paths):  # packed as layer_0 .. layer_{K-1}
            print(f"{path} exists. load checkpoint")
            ck = torch.load(path, map_location="cpu", weights_only=True)
            getattr(model, f"layer_{i}").load_state_dict(ck["0"])
        scaling_factor = a.n_train_step / a.n_test_step * a.hs_coeff_delta_h  # :626
        coeffs = [tuple([1.0 * a.hs_coeff_origin_h] + [1.0 * scaling_factor if j == k else 0.0 for j in range(K)])
                  for k in range(K)]
        model = model.to(self.device)
        if self.world > 1 and torch.distributed.is_initialized():
            broadcast_weights(model)
        if a.load_random_noise:
            pairs = self.random_noise_pairs(model, saved_noise=bool(getattr(a, "saved_random_noise", False)))
        else:
            pairs = self.precompute_pairs(model)
        return model, coeffs, pairs

    @torch.no_grad()
    def run_region_compose(self, spec):
        """--run_test --region_compose "a=classes b=classes ..": one image per latent in which every attribute edits
        only its own face-parsing region.  The K attributes run as rows of one batched trajectory (attribute-major,
        each with its own DeltaBlock, t_edit and t_addnoise, as --attr_sweep); after every step the K rows of an image
        are replaced by the per-pixel composite of the rows and the origin pass (UNetEngine.sample's compose).
        spec: region_compose_setup's result.  The composite is scored as one tuple (hs_coeff_origin_h, s, .., s)
        whose `attr` column joins the attributes with '+'."""
        from .face_parsing import FaceParser
        a = self.args
        print("Running Test (region composite)")
        attrs, classes, r, sigma, seg_sd, paths = spec
        exact = self.exact_inversion_setup()
        scorers = scoring.Scorers(self, ["+".join(attrs)])
        times = self.attr_sweep_schedules(attrs)  # prints each attribute's t_edit and t_addnoise
        self.compose_times = dict(zip(attrs, times))
        seq_test, seq_test_next = make_sequences(a.t_0, a.n_test_step)
        model, coeffs, pairs = self.attribute_run(paths)
        tuples = [tuple([coeffs[0][0]] + [coeffs[k][1 + k] for k in range(len(attrs))])]
        results = {}
        with scorers:  # --seg_consistency's parser serves the masks too
            compose = (scorers.nets.get("seg") or FaceParser(seg_sd, device=self.device), classes, r, sigma, times,
                       coeffs)
            for mode, step, x_lat, x0, ids, x0_source, anchors in self._edit_batches(model, pairs, scorers, exact):
                results[(mode, step)] = self.save_image(
                    model, x_lat, seq_test, seq_test_next, save_x0=a.save_x0, save_x_origin=a.save_x_origin,
                    x0_tensor=x0, folder_dir=a.test_image_folder, file_name=f'{mode}_{step}_{a.n_iter - 1}',
                    hs_coeff=tuples, scorers=scorers, mode=mode, batch_ids=ids, x0_source=x0_source,
                    region_compose=compose, **({"anchors": anchors} if exact else {}))
            scorers.finish(tuples)
            compose = None  # the parser goes with the scorers' networks, and the CUDA cache after it
        return results

    def compose_batch(self, model, x_lat, seq, seq_next, masks, ref, times, coeffs, anchors=None):
        """--region_compose's edit pass of one batch of B images: x_lat [B][C][S][S], masks [K][B][S][S] and the origin
        pass's trajectory ref [steps][B][C][S][S] on the device, times / coeffs per attribute.  Images run in chunks of
        b = --max_rows_per_replay // K (plan_compose) as K b rows, attribute-major, the last chunk padded, so that every
        chunk replays one graph.  The noise is one draw [n_stochastic][B][..] for the batch, each chunk's images
        repeated over its K rows (compose_noise).  anchors (--exact_inversion): the batch's inversion.Anchors; each chunk
        takes its images' anchors, padded as its latents are, and draws no noise.  Returns the composites [B][C][S][S]
        on the host."""
        eng = model.engine
        K, bs = masks.shape[0], x_lat.shape[0]
        b, chunks = plan_compose(bs, K, getattr(self.args, "max_rows_per_replay", 16))
        sch = self.sweep_schedule(seq, seq_next, [times[k] for k in range(K) for _ in range(b)],
                                  [coeffs[k] for k in range(K) for _ in range(b)])
        z = torch.randn((sch.n_stochastic, *x_lat.shape), device=eng.device) \
            if sch.n_stochastic and anchors is None else None
        per_image = lambda t, j0, j1: pad_rows(t[:, j0:j1].transpose(0, 1), b).transpose(0, 1)  # noqa: E731
        out = []
        for j0, j1 in chunks:
            kw = {"anchors": anchors.images(j0, j1, b)} if anchors is not None else {}
            x0 = self.edit_batch(model, pad_rows(x_lat[j0:j1], b).repeat(K, 1, 1, 1), sch,
                                 noise=compose_noise(z[:, j0:j1], b, K) if z is not None else None,
                                 compose=(per_image(masks, j0, j1), per_image(ref, j0, j1)), **kw)
            out.append(x0[:j1 - j0].clone())  # every attribute's row of an image holds its composite
        return torch.cat(out)

    def sweep_schedule(self, seq, seq_next, times, coeffs):
        """the RowSchedule of sweep rows: row r has t_edit / t_addnoise times[r] and coefficients coeffs[r], with the
        flags save_image's edit pass gives a single-attribute schedule (make_schedule)"""
        a = self.args
        return RowSchedule(self.betas, seq, seq_next, t_edit=[t[0] for t in times], t_addnoise=[t[1] for t in times],
                           hs_coeffs=coeffs, sample_type=getattr(a, "sample_type", "ddim"),
                           dt_lambda=getattr(a, "dt_lambda", 1.0), dt_end=999,
                           ignore_timestep=bool(getattr(a, "ignore_timesteps", False)), logvars=self.logvar)

    # ------------------------------------------------------------------------------------------
    def diff_style_setup(self):
        """--diff_style's requirements, checked before any model is loaded; raises ValueError with the reason.
        Returns (content image paths, style image paths, the hs_coeff values γ, one result per pair each)."""
        a = self.args
        if getattr(a, "run_test", False) or getattr(a, "lpips", False):
            raise ValueError("--diff_style is a mode of its own: it does not combine with --run_test or --lpips")
        if getattr(a, "user_defined_t_edit", None) is None:
            raise ValueError("--diff_style needs --user_defined_t_edit: DiffStyle edits with no text, so neither CLIP's "
                             "cosine nor the LPIPS tables can choose t_edit")
        if getattr(a, "sample_type", "ddim") != "ddim":
            raise ValueError(f"--diff_style needs --sample_type ddim, got {a.sample_type!r}: the reference's 'ddpm' step "
                             "never reads et_modified, so nothing would be injected")
        gammas = diff_style_gammas(getattr(a, "hs_coeff", 0.9), getattr(a, "hs_coeff_list", ""))
        paths = []
        for flag in ("content_dir", "style_dir"):
            d = getattr(a, flag, None)
            if not d or not os.path.isdir(d):
                raise ValueError(f"--diff_style: --{flag} {d!r} is not a directory")
            found = image_paths(d)
            if not found:
                raise ValueError(f"--diff_style: --{flag} {d!r} holds no png / jpg image")
            paths.append(found)
        names = {}
        for p in dict.fromkeys(paths[0] + paths[1]):
            c = diff_style_cache_path(self.config.data.category, a.n_inv_step, p)
            if names.setdefault(c, p) != p:
                raise ValueError(f"--diff_style: {names[c]!r} and {p!r} share the inversion cache {c!r} (the "
                                 "reference's name keeps the parent directory and the stem only)")
        return paths[0], paths[1], gammas

    @torch.no_grad()
    def precompute_pairs_with_h(self, model, img_paths):
        """[x0, 0, x_T, h_dic] of every image (diffusion_latent.py:877-947): DDIM inversion over
        zip(seq_inv_next[1:], seq_inv[1:]) with the plain UNet, h_dic[t] = the bottleneck h ([1,C,h,w] fp32) of the
        step that evaluated the UNet at t.  Cached on the CPU as precomputed/<category>_inv<n_inv_step>_<dir>_<stem>.pt
        in the reference's format; an existing cache (the reference's own included) is read unless --re_precompute.
        The images to invert run --bs_train per replay, h recorded inside the graph (UNetEngine.sample(record_h=True)).
        Under torchrun rank 0 inverts and writes the caches (temp file + rename), the other ranks load them after a
        barrier.  Returns {path: [x0, 0, x_T, h_dic]}; self.n_inverted counts the images inverted here."""
        a = self.args
        seq_inv, seq_inv_next = make_sequences(a.t_0, a.n_inv_step)
        os.makedirs('precomputed', exist_ok=True)
        out, todo = {}, []
        for p in dict.fromkeys(img_paths):
            cache = diff_style_cache_path(self.config.data.category, a.n_inv_step, p)
            if os.path.exists(cache) and not getattr(a, "re_precompute", False):
                out[p] = torch.load(cache, map_location="cpu", weights_only=True)
            else:
                todo.append((p, cache))
        self.n_inverted = 0
        if todo and self.rank == 0:
            eng = model.engine
            sch = Schedule.inversion(self.betas, seq_inv, seq_inv_next)
            bs = min(max(1, a.bs_train), len(todo))
            for k in range(0, len(todo), bs):  # every replay bs rows (the last one padded): one captured graph
                chunk = todo[k:k + bs]
                x0 = torch.cat([diff_style_image(p, self.config.data.image_size) for p, _ in chunk])
                x_lat = eng.sample(pad_rows(x0, bs).to(eng.device), sch, record_h=True).cpu()
                hs = eng.last_records["h"].cpu()
                for i, (p, cache) in enumerate(chunk):
                    h_dic = {int(st.t): hs[j][i:i + 1].clone() for j, st in enumerate(sch.steps)}
                    out[p] = [x0[i:i + 1].clone(), 0, x_lat[i:i + 1].clone(), h_dic]
                    _atomic_save(out[p], cache)
            self.n_inverted = len(todo)
        if todo and self.world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.barrier()
            for p, cache in todo:
                out.setdefault(p, torch.load(cache, map_location="cpu", weights_only=True))
        print(f"DiffStyle: {len(out)} images, {self.n_inverted} inverted, {len(out) - self.n_inverted} from cache")
        return out

    def diff_style_schedule(self, gamma):
        """the generation steps zip(reversed(seq_inv), reversed(seq_inv_next)) as the mode calls denoising_step:
        DDIM, t_edit = --user_defined_t_edit, eta = 1 below --t_noise, --dt_lambda from --dt_end on (save_image passes
        999 as dt_end; this mode passes --dt_end), hs_coeff = (γ,)"""
        a = self.args
        seq_inv, seq_inv_next = make_sequences(a.t_0, a.n_inv_step)
        return Schedule(self.betas, seq_inv, seq_inv_next, t_edit=a.user_defined_t_edit, t_addnoise=a.t_noise,
                        hs_coeff=(float(gamma),), sample_type="ddim", dt_lambda=a.dt_lambda, dt_end=a.dt_end)

    @torch.no_grad()
    def run_diff_style(self):
        """--diff_style: inject every content image's h into every style image's trajectory.  Row (content c, style s,
        γ) starts from the style's x_T and runs diff_style_schedule(γ) with delta_h = the content's h at each edit
        step: h2 = slerp(1 - γ, h, |h| h_c/|h_c|) (γ is forward's hs_coeff[0], so the weight on the content is 1 - γ).
        The content h at t_0, which the inversion never evaluates, is the bottleneck h of the content's x_T at t_0.
        Rows are (pair, γ), whole pairs per replay of at most --max_rows_per_replay rows; each row draws its own
        noise for the eta = 1 steps.  Writes <save_dir>/<content stem>__<style stem>.png: content x0, style x0, one
        result per γ; with --dino_structure also <save_dir>/diff_style_dino.tsv (scoring.write_diff_style_dino).  Returns {(content path, style path): results [len(γ)][3][S][S]}."""
        import torchvision.utils as tvu
        a = self.args
        self.prdc_check()
        self.edit_region_setup()  # refuses --diff_style
        self.region_compose_setup()  # refuses --diff_style
        self.exact_inversion_setup()  # refuses --diff_style
        if getattr(a, "content_preservation", False):
            self.content_preservation_setup()  # refuses --diff_style
        if getattr(a, "fid", False):
            self.fid_setup()  # refuses --diff_style, before any model loads
        dino_sd = self.dino_structure_setup() if getattr(a, "dino_structure", False) else None
        contents, styles, gammas = self.diff_style_setup()
        print(f"DiffStyle: hs_coeff {gammas} (slerp weight on the content h: 1 - hs_coeff)")
        model = self.load_pretrained_model().to(self.device)
        if self.world > 1 and torch.distributed.is_initialized():
            broadcast_weights(model)
        eng = model.engine
        cached = self.precompute_pairs_with_h(model, contents + styles)
        sch = self.diff_style_schedule(gammas[0])
        t0 = sch.steps[0].t
        # content h at t_0: one plain UNet evaluation of each content's x_T
        h_c = {}
        bs = min(max(1, a.bs_train), len(contents))
        for k in range(0, len(contents), bs):
            chunk = contents[k:k + bs]
            x_T = pad_rows(torch.cat([cached[p][2] for p in chunk]), bs).to(eng.device)
            mid = eng.forward(x_T, torch.full((bs,), float(t0), device=eng.device))[3].cpu()
            for i, p in enumerate(chunk):
                h_c[p] = dict(cached[p][3])
                h_c[p][t0] = mid[i:i + 1].clone()
        pairs = [(c, s_) for c in contents for s_ in styles]
        ppc, chunks = plan_sweep(len(pairs), len(gammas), getattr(a, "max_rows_per_replay", 16))
        R = ppc * len(gammas)
        edit_ts = [st.t for st in sch.steps if st.edit]
        print(f"DiffStyle: {len(pairs)} pairs, {len(pairs) * len(gammas)} rows, {len(chunks)} replays of {R} rows")
        os.makedirs(a.save_dir, exist_ok=True)
        results = {}
        dino, dino_rows = None, []
        if dino_sd is not None:
            from .dino import DINO
            dino = DINO(dino_sd, device=self.device)
            dino_sd = None
        for ci, chunk in enumerate(chunks):
            if ci % self.world != self.rank:  # chunks sharded round-robin across ranks
                continue
            rows = [(pairs[q], g) for q in chunk for g in gammas]
            rows += [rows[-1]] * (R - len(rows))
            x_T = torch.cat([cached[s_][2] for (_, s_), _ in rows])
            kw = {"hs_coeffs": torch.tensor([[g] for _, g in rows], dtype=torch.float32), "use_mask": bool(a.use_mask)}
            if edit_ts:
                kw["delta_hs"] = diff_style_delta_hs([h_c[c] for (c, _), _ in rows], edit_ts)
            noise = None
            if sch.n_stochastic:  # one draw per row, made on the device up front
                noise = torch.cat([torch.randn((sch.n_stochastic, 1, *x_T.shape[1:]), device=eng.device)
                                   for _ in range(len(chunk) * len(gammas))], dim=1)
                noise = pad_rows(noise.transpose(0, 1), R).transpose(0, 1).contiguous()
            x0 = self.edit_batch(model, x_T, sch, noise=noise, **kw)
            for j, q in enumerate(chunk):
                c, s_ = pairs[q]
                res = x0[j * len(gammas):(j + 1) * len(gammas)].clone()
                results[(c, s_)] = res
                grid = (torch.cat([cached[c][0].cpu(), cached[s_][0].cpu(), res]) + 1) * 0.5
                tvu.save_image(tvu.make_grid(grid, nrow=grid.shape[0], padding=1),
                               os.path.join(a.save_dir, f"{_stem(c)}__{_stem(s_)}.png"))
                if dino is not None:  # each result against the content and the style x0
                    sc, ss = dino.scores(cached[c][0], res)[:, 0], dino.scores(cached[s_][0], res)[:, 0]
                    dino_rows += [(c, s_, g, *sc[k, 0:1].tolist(), *ss[k, 0:1].tolist(), *sc[k, 1:].tolist(),
                                   *ss[k, 1:].tolist()) for k, g in enumerate(gammas)]
        if dino is not None:
            dino = None
            torch.cuda.empty_cache()
            rows = scoring.gather_rows(self, dino_rows)
            if rows is not None:
                self.diff_style_dino = scoring.write_diff_style_dino(os.path.join(a.save_dir, "diff_style_dino.tsv"),
                                                                     rows)
        return results


def diff_style_gammas(hs_coeff, hs_coeff_list):
    """the hs_coeff values of a --diff_style run: --hs_coeff_list ("0.9 0.7 0.5"), else [--hs_coeff]"""
    if not hs_coeff_list:
        return [float(hs_coeff)]
    if float(hs_coeff) != 0.9:
        raise ValueError(f"--diff_style: give either --hs_coeff ({hs_coeff}) or --hs_coeff_list, not both")
    try:
        gammas = [float(v) for v in str(hs_coeff_list).split()]
    except ValueError:
        raise ValueError(f"--hs_coeff_list {hs_coeff_list!r} is not a list of numbers") from None
    if not gammas:
        raise ValueError("--hs_coeff_list names no value")
    return gammas


def h_direction_coeffs(a):
    """the hs_coeff tuples of --run_test --h_direction: (--hs_coeff_origin_h, α) with α = --hs_coeff_delta_h as given
    (no n_train_step / n_test_step scaling: a direction has no training grid); --delta_interpolation: (1, v α) for v
    in linspace(--min_delta, --max_delta, --num_delta)"""
    alpha = float(a.hs_coeff_delta_h)
    if a.delta_interpolation:
        return [(1.0, v * alpha) for v in np.linspace(a.min_delta, a.max_delta, a.num_delta).tolist()]
    return (1.0 * a.hs_coeff_origin_h, alpha)


def image_paths(folder):
    """every png / jpg of a directory, sorted"""
    return sorted(os.path.join(folder, f) for f in os.listdir(folder) if f.lower().endswith((".png", ".jpg", ".jpeg")))


def diff_style_cache_path(category, n_inv_step, img_path):
    """precompute_pairs_with_h's cache file (diffusion_latent.py:883-885), the reference's expression kept as is: the
    last two '/'-parts of the text before the path's last dot ("c/x.png" -> c_x; a dot in a directory name cuts the
    directories before it, "a.b/c/x.png" -> c_x, and a dotted stem keeps its last part only, "c/x.v1.png" -> v1)"""
    name = "_".join(img_path.split(".")[-2].split('/')[-2:])
    return os.path.join('precomputed', category + '_inv' + str(n_inv_step) + '_' + name + '.pt')


def diff_style_image(path, size):
    """precompute_pairs_with_h's transform (:896-906): centre crop to the shorter side, Resize((size, size)),
    ToTensor, Normalize(0.5, 0.5) -> [1,3,size,size] in [-1, 1]"""
    from PIL import Image
    from torchvision import transforms
    image = Image.open(path).convert('RGB')
    image = transforms.CenterCrop(min(image.size))(image)
    tf = transforms.Compose([transforms.Resize((size, size)), transforms.ToTensor(),
                             transforms.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
    return tf(image)[None]


def diff_style_delta_hs(h_dics, edit_ts):
    """delta_hs of UNetEngine.sample for rows with their own content h: [edit steps][rows][C][h][w], row r's h_dics[r][t]
    at every edit step t"""
    out = []
    for t in edit_ts:
        missing = [r for r, d in enumerate(h_dics) if int(t) not in d]
        if missing:
            raise KeyError(f"DiffStyle: no content h at edit step t={t} (rows {missing})")
        out.append(torch.cat([d[int(t)].float() for d in h_dics]))
    return torch.stack(out)


def _stem(path):
    return os.path.splitext(os.path.basename(path))[0]


def sweep_rows(chunk, tpc, bs):
    """the attribute of every trajectory row of one sweep chunk: attribute-major (attribute, image) rows, padded to
    tpc * bs rows with the last attribute (padding rows are discarded)"""
    rows = [k for k in chunk for _ in range(bs)]
    return rows + [rows[-1]] * (tpc * bs - len(rows))


def plan_sweep(n_tuples, bs, max_rows):
    """Chunks of an hs_coeff sweep run as rows of one batch: (tuples per chunk, [tuple indices of each chunk]).
    A chunk holds whole tuples, at most max_rows // bs of them (at least one); every chunk runs as tuples-per-chunk * bs
    rows, the last one padded (pad_rows), so that one plan and one captured graph serve them all."""
    tpc = min(n_tuples, max(1, max_rows // bs))
    return tpc, [list(range(k, min(k + tpc, n_tuples))) for k in range(0, n_tuples, tpc)]


def read_text_dic(path):
    """SRC_TRG_TXT_DIC of the reference's utils/text_dic.py: the literal assigned to that name, read with ast (the
    file is parsed, never imported or executed)"""
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found: pass --text_dic <file defining SRC_TRG_TXT_DIC> (the reference's "
                                "utils/text_dic.py)")
    with open(path, encoding="utf-8") as f:
        tree = ast.parse(f.read(), filename=path)
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "SRC_TRG_TXT_DIC"
                                                for t in node.targets):
            return ast.literal_eval(node.value)
    raise ValueError(f"{path} assigns no SRC_TRG_TXT_DIC literal")


def lpips_tables(seq_inv, seq_inv_next, per_image):
    """The four TSV texts of compute_lpips_distance (diffusion_latent.py:1224-1298) from per-image, per-step distances:
    per_image[i] = (LPIPS(x_t, x0) per step, LPIPS(x0_t, x0) per step) over the steps zip(seq_inv_next[1:],
    seq_inv[1:]), each value keyed by the step's t_next.  One row "<t><TAB><value>" per t in seq_inv[1:].  A t that occurs
    twice in seq_inv collects the values of both its steps and is written twice, the second time with the same mean
    and std 0: the reference's loop replaces each list by its mean on the first visit."""
    lx = {s: [] for s in seq_inv[1:]}
    lx0 = {s: [] for s in seq_inv[1:]}
    for vx, vx0 in per_image:
        for it, (_, j) in enumerate(zip(seq_inv_next[1:], seq_inv[1:])):
            lx[j].append(vx[it])
            lx0[j].append(vx0[it])
    sx, sx0 = {}, {}
    out = {"x": "", "x_std": "", "x0_t": "", "x0_t_std": ""}
    for seq in seq_inv[1:]:
        sx[seq] = np.std(lx[seq])
        lx[seq] = np.mean(lx[seq])
        sx0[seq] = np.std(lx0[seq])
        lx0[seq] = np.mean(lx0[seq])
        out["x"] += f"{seq}\t{lx[seq]}\n"
        out["x_std"] += f"{seq}\t{sx[seq]}\n"
        out["x0_t"] += f"{seq}\t{lx0[seq]}\n"
        out["x0_t_std"] += f"{seq}\t{sx0[seq]}\n"
    return out


def plan_compose(bs, K, max_rows):
    """Chunks of a --region_compose batch of bs images with K attributes: (b, [(first, end) image range of each
    chunk]).  A chunk holds b = min(bs, max_rows // K) images (at least one) and runs as K b rows; the last one is
    padded (pad_rows), so that every chunk replays one graph."""
    b = min(bs, max(1, max_rows // K))
    return b, [(j, min(j + b, bs)) for j in range(0, bs, b)]


def compose_noise(z, b, K):
    """the noise of one --region_compose chunk, [n_stochastic][K b][...], from the batch's draw of its images z
    [n_stochastic][m <= b][...]: padded to b images (padding copies the last image), then repeated over the K
    attribute rows, so that the K rows of an image share its noise"""
    if z.shape[1] < b:
        z = torch.cat([z, z[:, -1:].expand(z.shape[0], b - z.shape[1], *z.shape[2:])], dim=1)
    return z.repeat(1, K, *([1] * (z.dim() - 2)))


def pad_rows(t, n):
    """t with its last row repeated up to n rows (padding rows of a sweep chunk; their results are discarded)"""
    if t.shape[0] >= n:
        return t
    return torch.cat([t, t[-1:].expand(n - t.shape[0], *t.shape[1:])], dim=0)


def chunk_noise(n_tuples, tpc, bs, draw):
    """Noise of one sweep chunk, [n_stochastic][tpc * bs][...]: draw() ([n_stochastic][bs][...]) once per tuple, in tuple
    order, concatenated along the batch axis, so the random stream is consumed exactly as by one replay per tuple.
    Padding rows copy the last real row and draw nothing."""
    z = torch.cat([draw() for _ in range(n_tuples)], dim=1)
    if n_tuples < tpc:
        pad = (tpc - n_tuples) * bs
        z = torch.cat([z, z[:, -1:].expand(z.shape[0], pad, *z.shape[2:])], dim=1)
    return z


def _atomic_save(obj, path):
    """write to a temp file in the same directory, then rename: a concurrent reader never sees a truncated cache"""
    tmp = f"{path}.tmp.{os.getpid()}"
    torch.save(obj, tmp)
    os.replace(tmp, path)


def broadcast_weights(model, src=0):
    """the one collective of the path: rank `src`'s parameters to every rank (NCCL over NVLink), as one flat buffer"""
    import torch.distributed as dist
    params = [p for p in model.parameters()]
    flat = torch.cat([p.detach().reshape(-1) for p in params])
    dist.broadcast(flat, src=src)
    off = 0
    for p in params:
        n = p.numel()
        p.data.copy_(flat[off:off + n].view_as(p))
        off += n
    model.refresh_weights()


def _load_image_folder(folder, size, limit):
    from PIL import Image
    names = sorted(f for f in os.listdir(folder) if f.lower().endswith((".png", ".jpg", ".jpeg")))[:limit]
    out = []
    for f in names:
        im = Image.open(os.path.join(folder, f)).convert("RGB").resize((size, size), Image.BICUBIC)
        t = torch.from_numpy(np.asarray(im).copy()).permute(2, 0, 1).float() / 255.0
        out.append((t * 2.0 - 1.0)[None])  # rescaled to [-1, 1] (config.data.rescaled)
    return out


def _read_tsv(path):
    rows = []
    with open(path) as f:
        for line in f:
            parts = line.strip().split("\t")
            if len(parts) >= 2:
                try:
                    rows.append((int(float(parts[0])), float(parts[1])))
                except ValueError:
                    continue
    return sorted(rows)
