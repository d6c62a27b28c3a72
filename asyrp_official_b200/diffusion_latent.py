"""`Asyrp` runner — inference/editing half of the reference's diffusion_latent.py on the CUDA engine.

Mirrors, with the same attribute / flag names:
  Asyrp.__init__               diffusion_latent.py:32-73    betas, logvar tables
  Asyrp.load_pretrained_model  :76-126                      dataset -> UNet family dispatch, load_state_dict(strict=False)
  Asyrp.run_test               :547-874                     sequences, Δh checkpoint, hs_coeff (single / multi-attribute /
                                                            interpolation sweep), batching of latents
  Asyrp.save_image             :445-544                     the reverse loops + PNG grid
  Asyrp.random_noise_pairs     :1087-1188                   x_T = N(0,1) per image
  Asyrp.set_t_edit_t_addnoise  :1308-1416                   user-defined values or LPIPS-table lookup given a cosine

Differences (documented in INTEGRATION.md): the reverse loop is UNetEngine.sample() — one CUDA graph per
(batch, schedule) instead of 40 Python iterations; pretrained weights come from --model_path (no URL download);
CLIP is not available, so t_edit / t_addnoise come from --user_defined_t_edit/_t_addnoise or from the shipped
LPIPS tables with an explicit --clip_cosine.  With torch.distributed initialised (one process per GPU) the image
batches are sharded round-robin across ranks; the only collective is the initial weight broadcast.
"""
import os
import time

import numpy as np
import torch

from .modules import DDPM, guided_Diffusion, i_DDPM
from .schedule import Schedule
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
        similarity in the reference (:1319-1329); CLIP is unavailable offline, so it is the explicit --clip_cosine.
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
        if not os.path.exists(p0) or (ut is None and cosine is None):
            raise ValueError(f"t_edit / t_addnoise undefined: pass --user_defined_t_edit and --user_defined_t_addnoise, "
                             f"or --clip_cosine with --lpips_table_dir (looked for {p0}; CLIP is not available offline)")
        table = _read_tsv(p0)
        self.t_edit = ut if ut is not None else next(t for t, v in table if v >= LPIPS_th * cosine)
        if ua is not None:
            self.t_addnoise = ua
        else:
            if getattr(a, "add_noise_from_xt", False):
                table = _read_tsv(os.path.join(tdir, f"{name}_LPIPS_distance_x.tsv"))
            self.t_addnoise = next(t for t, v in table if v >= LPIPS_addnoise_th)
        return cosine

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
    def invert_batch(self, model, x0, n_inv_step=None):
        """DDIM inversion x_0 -> x_T followed by the reconstruction x_T -> x_rec with --sample_type, both as graph
        replays (precompute_pairs, diffusion_latent.py:1028-1072).  Returns (x_T, x_rec) on the host."""
        a = self.args
        n = n_inv_step or a.n_inv_step
        seq_inv = [int(s + 1e-6) for s in list(np.linspace(0, 1, n) * a.t_0)]
        seq_inv_next = [-1] + list(seq_inv[:-1])
        eng = model.engine
        x_lat = eng.sample(x0.to(eng.device), Schedule.inversion(self.betas, seq_inv, seq_inv_next))
        sch = Schedule(self.betas, seq_inv, seq_inv_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False,
                       sample_type=getattr(a, "sample_type", "ddim"), logvars=self.logvar)
        noise = torch.randn((sch.n_stochastic, *x_lat.shape), device=eng.device) if sch.n_stochastic else None
        x_rec = eng.sample(x_lat, sch, noise=noise)
        return x_lat.cpu(), x_rec.cpu()

    @torch.no_grad()
    def precompute_pairs(self, model, save_imgs=False):
        """[x0, x_rec, x_T] triples per image, cached as precomputed/<category>_<mode>_t<t_0>_nim<N>_ninv<k>_pairs.pth
        — the reference's file name and list-of-triples format (:974-982,1072,1082).  Images come from
        --custom_train_dataset_dir / --custom_test_dataset_dir (png/jpg, resized to image_size, scaled to [-1, 1]);
        the reference's LMDB dataset classes are out of scope.  Under torchrun rank 0 inverts and writes the cache
        (temp file + rename), the other ranks load it after a barrier."""
        a, out = self.args, {}
        os.makedirs('precomputed', exist_ok=True)
        for mode, n in (("train", a.n_train_img), ("test", a.n_test_img)):
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
        ([n_stochastic, B, 3, S, S]) is given.  sample_kw: delta_hs / use_mask / record_dh / record_process of
        UNetEngine.sample()."""
        eng = model.engine
        dev = eng.device
        if schedule.n_stochastic and noise is None:
            noise = torch.randn((schedule.n_stochastic, *x_lat.shape), device=dev)
        elif noise is not None:
            noise = noise.to(dev, non_blocking=True)
        x0 = eng.sample(x_lat.to(dev, non_blocking=True), schedule, noise=noise, **sample_kw)
        if out is not None:
            out.copy_(x0, non_blocking=True)
            return out
        return x0.cpu()

    def _write_process(self, eng, schedule, folder, prefix, bs):
        """per-step grids of [x_t ; x0_t] (save_process_origin / save_process_delta_h, :485-491,523-527)"""
        import torchvision.utils as tvu
        rec = eng.last_records
        os.makedirs(folder, exist_ok=True)
        for k, st in enumerate(schedule.steps):
            out = (torch.cat([rec["x"][k], rec["x0_t"][k]], dim=0).cpu() + 1) * 0.5
            tvu.save_image(tvu.make_grid(out, nrow=bs, padding=1), os.path.join(folder, f'{prefix}_{int(st.t)}.png'))

    @torch.no_grad()
    def save_image(self, model, x_lat_tensor, seq_inv, seq_inv_next, save_x0=False, save_x_origin=False,
                   save_process_delta_h=False, save_process_origin=False, x0_tensor=None, delta_h_dict=None,
                   get_delta_hs=False, folder_dir="", file_name="", hs_coeff=(1.0, 1.0)):
        """rows of the grid: [x0] [origin DDIM] one row per hs_coeff tuple  (diffusion_latent.py:445-544).

        delta_h_dict: {t: None | Δh tensor}.  Entries that are tensors select the explicit-Δh branch for that step
        (raw-Δh checkpoints, mean Δh); get_delta_hs: run the DeltaBlocks and ADD their per-step output into
        delta_h_dict (mean-Δh extraction, :528-532)."""
        import torchvision.utils as tvu
        a = self.args
        time_s = time.time()
        eng = model.engine
        bs = x_lat_tensor.shape[0]
        x_list = []
        if save_x0 and x0_tensor is not None:
            x_list.append(x0_tensor.cpu())
        if save_x_origin:
            sch = self.make_schedule(seq_inv, seq_inv_next, (1.0,), edit=False,
                                     addnoise=bool(getattr(a, "origin_process_addnoise", False)))
            x_list.append(self.edit_batch(model, x_lat_tensor, sch, record_process=save_process_origin))
            if save_process_origin:
                self._write_process(eng, sch, os.path.join(folder_dir, file_name), "origin", bs)
        if not getattr(a, "pass_editing", False):
            coeffs = hs_coeff if isinstance(hs_coeff, list) else [hs_coeff]
            for tup in coeffs:
                sch = self.make_schedule(seq_inv, seq_inv_next, tup)
                edit_ts = [st.t for st in sch.steps if st.edit and st.kind == "ddim"]
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
                x_list.append(self.edit_batch(model, x_lat_tensor, sch, record_process=save_process_delta_h, **kw))
                if save_process_delta_h:
                    self._write_process(eng, sch, os.path.join(folder_dir, file_name), "delta_h", bs)
                if get_delta_hs:
                    rec = eng.last_records["delta_h"].cpu()
                    for ei, t in enumerate(edit_ts):
                        delta_h_dict[int(t)] = rec[ei] if delta_h_dict.get(int(t)) is None else delta_h_dict[int(t)] + rec[ei]
        x = (torch.cat(x_list, dim=0) + 1) * 0.5
        grid = tvu.make_grid(x, nrow=a.bs_train, padding=1)
        os.makedirs(folder_dir, exist_ok=True)
        path = os.path.join(folder_dir, f'{file_name}_ngen{a.n_train_step}.png')
        tvu.save_image(grid, path)
        print(f'{time.time() - time_s} seconds, {file_name}_ngen{a.n_train_step}.png is saved')
        return x_list

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def run_test(self):
        a = self.args
        print("Running Test")
        if getattr(a, "warigari", 0.0):
            print("--warigari is accepted and has no effect (the reference's branch returns the same values, "
                  "utils/diffusion_utils.py:103-109)")
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
        if a.multiple_attr:
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
        if os.path.exists(save_name_list[0]):
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
        if a.delta_interpolation:  # :726-755
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
        target_ids = None
        if getattr(a, "target_image_id", None):
            target_ids = [int(i) for i in str(a.target_image_id).split(" ")]
            assert a.bs_train == 1, "target_image_id is only supported for batch_size == 1"
        results = {}
        try:
            for mode, do, n_img in (("train", a.do_train, a.n_train_img), ("test", a.do_test, a.n_test_img)):
                if not do:
                    continue
                x_lat_tensor, x0_tensor, batch_idx = None, None, 0
                for step, (x0, _, x_lat) in enumerate(pairs[mode]):
                    if target_ids is not None and step not in target_ids:
                        continue
                    if a.start_image_id > step:
                        continue
                    x_lat_tensor = x_lat if x_lat_tensor is None else torch.cat((x_lat_tensor, x_lat), dim=0)
                    if a.use_x0_tensor:
                        x0_tensor = x0 if x0_tensor is None else torch.cat((x0_tensor, x0), dim=0)
                    if (step + 1) % a.bs_train != 0:
                        continue
                    if batch_idx % self.world == self.rank:  # batch-sharded across ranks, no per-step communication
                        results[(mode, step)] = self.save_image(
                            model, x_lat_tensor, seq_test, seq_test_next, save_x0=a.save_x0,
                            save_x_origin=a.save_x_origin, x0_tensor=x0_tensor, delta_h_dict=delta_h_dict,
                            get_delta_hs=bool(num_mean),
                            save_process_origin=bool(getattr(a, "save_process_origin", False)),
                            save_process_delta_h=bool(getattr(a, "save_process_delta_h", False)),
                            folder_dir=a.test_image_folder, file_name=f'{mode}_{step}_{a.n_iter - 1}', hs_coeff=hs_coeff)
                    batch_idx += 1
                    if step == n_img - 1:
                        break
                    if mode == "train" and num_mean and step == num_mean - 1:
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
                    x_lat_tensor, x0_tensor = None, None
        finally:
            a.train_delta_h = a_train_delta_h_prev
        self.last_delta_h_dict = delta_h_dict
        return results


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
