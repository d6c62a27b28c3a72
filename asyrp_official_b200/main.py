"""CLI of the editing / inference path: the flags of the reference's main.py that reach `Asyrp.run_test`
(SURVEY.md Appendix E), same names and defaults (main.py:12-229), same experiment-directory naming (:235).

    python -m asyrp_official_b200.main --run_test --config celeba.yml --exp ./runs/smiling --edit_attr smiling \
        --train_delta_block --get_h_num 1 --load_random_noise --user_defined_t_edit 500 --user_defined_t_addnoise 200 \
        --manual_checkpoint_name smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth --model_path celeba_hq.ckpt \
        --n_test_img 32 --bs_train 16 --n_test_step 40 --n_train_step 40

DiffStyle content injection (main.py:192-202; the loop is this build's composition of the reference's functions):

    python -m asyrp_official_b200.main --diff_style --config celeba.yml --model_path celeba_hq.ckpt \
        --content_dir content --style_dir style --save_dir results --user_defined_t_edit 400 \
        --hs_coeff_list "0.9 0.7 0.5" --t_noise 200 --dt_lambda 0.9985 --dt_end 950 --bs_train 8

Multi-GPU: launch with torchrun (one process per GPU); image batches are sharded across ranks.
"""
import argparse
import logging
import os
import sys
import traceback

import numpy as np
import torch

from .configs import load_config


def build_parser():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sa = dict(action='store_true')
    p.add_argument('--sh_file_name', type=str, default='script.sh')
    p.add_argument('--user_defined_t_edit', type=int)
    p.add_argument('--user_defined_t_addnoise', type=int)
    p.add_argument('--lpips_edit_th', type=float, default=0.33)
    p.add_argument('--lpips_addnoise_th', type=float, default=0.1)
    p.add_argument('--add_noise_from_xt', **sa)
    p.add_argument('--origin_process_addnoise', **sa)
    p.add_argument('--run_test', **sa)
    p.add_argument('--lpips', **sa)
    p.add_argument('--train_delta_block', **sa)
    p.add_argument('--train_delta_h', **sa)
    p.add_argument('--ignore_timesteps', **sa)
    p.add_argument('--use_x0_tensor', **sa)
    p.add_argument('--save_x0', **sa)
    p.add_argument('--save_x_origin', **sa)
    p.add_argument('--load_random_noise', **sa)
    p.add_argument('--saved_random_noise', **sa)
    p.add_argument('--delta_interpolation', **sa)
    p.add_argument('--max_delta', type=float, default=1.0)
    p.add_argument('--min_delta', type=float, default=0.0)
    p.add_argument('--num_delta', type=int, default=5)
    p.add_argument('--hs_coeff_delta_h', type=float, default=1.0)
    p.add_argument('--hs_coeff_origin_h', type=float, default=1.0)
    p.add_argument('--target_image_id', type=str)
    p.add_argument('--start_image_id', type=int, default=0)
    p.add_argument('--save_process_origin', **sa)
    p.add_argument('--save_process_delta_h', **sa)
    p.add_argument('--num_mean_of_delta_hs', type=int, default=0)
    p.add_argument('--multiple_attr', type=str, default='')
    p.add_argument('--multiple_hs_coeff', type=str, default='')
    p.add_argument('--manual_checkpoint_name', type=str, default="")
    p.add_argument('--choose_checkpoint_num', type=str, default='')
    p.add_argument('--load_from_checkpoint', type=str)
    p.add_argument('--pass_editing', **sa)
    p.add_argument('--DirectionalClipSmilarity', **sa)
    p.add_argument('--warigari', type=float, default=0.0)
    p.add_argument('--config', type=str, required=True)
    p.add_argument('--seed', type=int, default=1234)
    p.add_argument('--exp', type=str, default='./runs/')
    p.add_argument('--verbose', type=str, default='info')
    p.add_argument('--ni', type=int, default=1)
    p.add_argument('--edit_attr', type=str, default=None)
    p.add_argument('--src_txts', type=str, action='append')
    p.add_argument('--trg_txts', type=str, action='append')
    p.add_argument('--t_0', type=int, default=999)
    p.add_argument('--n_inv_step', type=int, default=40)
    p.add_argument('--n_train_step', type=int, default=6)
    p.add_argument('--n_test_step', type=int, default=40)
    p.add_argument('--sample_type', type=str, default='ddim')
    p.add_argument('--do_train', type=int, default=1)
    p.add_argument('--do_test', type=int, default=1)
    p.add_argument('--bs_train', type=int, default=1)
    p.add_argument('--n_train_img', type=int, default=50)
    p.add_argument('--n_test_img', type=int, default=10)
    p.add_argument('--model_path', type=str, default=None)
    p.add_argument('--get_h_num', type=int, default=0)
    p.add_argument('--re_precompute', **sa)
    p.add_argument('--custom_train_dataset_dir', type=str, default="./custom/train")
    p.add_argument('--custom_test_dataset_dir', type=str, default="./custom/test")
    p.add_argument('--dt_lambda', type=float, default=1.0)
    p.add_argument('--dt_end', type=int, default=950)
    # DiffStyle (main.py:192-202)
    p.add_argument('--diff_style', **sa)
    p.add_argument('--content_dir', type=str, default="./source_images/content")
    p.add_argument('--style_dir', type=str, default="./source_images/style")
    p.add_argument('--save_dir', type=str, default="./results")
    p.add_argument('--hs_coeff', type=float, default=0.9)
    p.add_argument('--use_mask', **sa)
    p.add_argument('--t_noise', type=int, default=0)
    p.add_argument('--n_iter', type=int, default=1)
    # additions of this build (documented in INTEGRATION.md)
    p.add_argument('--synthetic_weights', **sa, help='seeded random UNet weights instead of --model_path')
    p.add_argument('--clip_cosine', type=float, help='text-direction cosine to use instead of computing it with CLIP')
    p.add_argument('--clip_weights', type=str, default=None,
                   help="CLIP's model file (e.g. ~/.cache/clip/ViT-B-16.pt, or a torch.save of its state dict): the "
                        "text tower computes the cosine that picks t_edit")
    p.add_argument('--clip_vocab', type=str, default=None,
                   help="CLIP's bpe_simple_vocab_16e6.txt.gz (inside the installed clip package)")
    p.add_argument('--text_dic', type=str, default=None,
                   help='file defining SRC_TRG_TXT_DIC, read with ast (default utils/text_dic.py)')
    p.add_argument('--text_templates', type=str, default=None,
                   help='file defining imagenet_templates, read with ast, for --DirectionalClipSmilarity (default '
                        'utils/text_templates.py)')
    p.add_argument('--id_similarity', **sa,
                   help='--run_test: score every edit for identity preservation, 1 - IDLoss (ArcFace IR-SE50) against '
                        'the unedited DDIM pass of the same x_T, written next to the PNG')
    p.add_argument('--id_weights', type=str, default='pretrained/model_ir_se50.pth',
                   help="the reference's ArcFace weights (MODEL_PATHS['ir_se50']) for --id_similarity")
    p.add_argument('--seg_consistency', **sa,
                   help='--run_test: score every edit for segmentation consistency, the fraction of 512 x 512 pixels '
                        'whose face-parsing BiSeNet label equals that of the unedited DDIM pass of the same x_T, '
                        'written next to the PNG')
    p.add_argument('--seg_weights', type=str, default='pretrained/79999_iter.pth',
                   help='torch.save of the face-parsing BiSeNet(n_classes=19) state dict for --seg_consistency')
    p.add_argument('--fid', **sa,
                   help='--run_test: score each set of edits (one per hs_coeff tuple or --attr_sweep attribute) for '
                        'realism with FID and KID on Inception-v3 pool features against the unedited DDIM pass of '
                        'the same x_T, written to <test_image_folder>/<mode>_ngen<n_train_step>_fid.tsv')
    p.add_argument('--fid_weights', type=str, default='pretrained/pt_inception-2015-12-05-6726825d.pth',
                   help="pytorch-fid's FID Inception-v3 weights for --fid")
    p.add_argument('--fid_ref', type=str, default=None,
                   help='--fid: also score the origin set and each set of edits against the reference statistics of '
                        'real images in this .npz (python -m asyrp_official_b200.fid --save-stats DIR OUT.npz), '
                        'written to <test_image_folder>/<mode>_ngen<n_train_step>_fid_real.tsv')
    p.add_argument('--kid_subsets', type=int, default=100,
                   help='--fid_ref: random subsets of the subset KID (KID_mean / KID_std); 0 = none')
    p.add_argument('--kid_subset_size', type=int, default=1000,
                   help='--fid_ref: rows per subset of the subset KID (a set smaller than this gets nan)')
    p.add_argument('--prdc', **sa,
                   help='--fid: also score each set of edits with improved precision / recall and density / coverage '
                        'from k-nearest-neighbour balls of the pool features, against the origin set '
                        '(<mode>_ngen<n_train_step>_prdc.tsv) and with --fid_ref against its features (_prdc_real.tsv)')
    p.add_argument('--prdc_k', type=int, default=5,
                   help='--prdc: the k of the k-nearest-neighbour balls, 1..32 (a set of k images or fewer gets nan)')
    p.add_argument('--lpips_table_dir', type=str,
                   help='directory with <config stem>_LPIPS_distance_{x,x0_t}.tsv (read by --run_test, written by '
                        '--lpips; default utils)')
    p.add_argument('--lpips_weights', type=str, default=None,
                   help="torch.save of the lpips package's LPIPS(net='alex').state_dict() (--lpips, "
                        "--content_preservation)")
    p.add_argument('--content_preservation', **sa,
                   help='--run_test: score every edit for content preservation, PSNR, SSIM, MS-SSIM and LPIPS-Alex '
                        '(--lpips_weights, or seeded weights with --synthetic_weights) of the saved u8 image against '
                        'the unedited DDIM pass of the same x_T, and that pass against the input image for latents '
                        'inverted from images, written next to the PNG (images larger than 160 x 160)')
    p.add_argument('--dino_structure', **sa,
                   help='--run_test: score every edit against the unedited DDIM pass of the same x_T (and that pass '
                        'against the input image for latents inverted from images) with DINO-ViT: the key '
                        'self-similarity structure distance and the CLS cosine, written next to the PNG; '
                        '--diff_style: score every result against its content and its style image, written to '
                        '<save_dir>/diff_style_dino.tsv')
    p.add_argument('--dino_weights', type=str, default='pretrained/dino_vitbase8_pretrain.pth',
                   help="torch.save of DINO's VisionTransformer state dict (ViT-S/8, S/16, B/8 or B/16) for "
                        "--dino_structure")
    p.add_argument('--checkpoint_dir', type=str, default='checkpoint')
    p.add_argument('--max_rows_per_replay', type=int, default=16,
                   help='rows (hs_coeff tuples x images) of one batched trajectory in save_image; bounds the memory of '
                        'the per-batch plan (DDPM 256x256: about 4.3 GB at 16 rows); 1 = one replay per tuple')
    p.add_argument('--hs_coeff_list', type=str, default='',
                   help='--diff_style: several hs_coeff values ("0.9 0.7 0.5"), one result per value for every '
                        'content / style pair, run as rows of one batch')
    p.add_argument('--attr_sweep', type=str, default='',
                   help='--run_test: edit every image with each of these attributes ("smiling angry young"), one grid '
                        'row per attribute, each row what --edit_attr <attribute> gives with its own t_edit / '
                        't_addnoise; the checkpoint name\'s "attribute" is replaced by each attribute')
    p.add_argument('--h_directions', **sa,
                   help='find editing directions from the statistics of the bottleneck h over many samples, with '
                        'forward passes only (per-timestep PCA with --h_pca, or a mean difference with --h_pos_dir / '
                        '--h_neg_dir); writes pc<k>.pth or mean_diff.pth and h_directions.tsv to --h_direction_out')
    p.add_argument('--h_pca', type=int, default=None,
                   help='--h_directions: the top K principal components of h over the n_train_img "train" latents '
                        'of --run_test (--load_random_noise, or --custom_train_dataset_dir images inverted and cached '
                        'by the same precompute step); 1 <= K <= n - 1')
    p.add_argument('--h_pos_dir', type=str, default=None,
                   help='--h_directions: images showing the attribute, the first --n_train_img of them by name, '
                        'DDIM-inverted; the direction is the mean h of these minus the mean h of --h_neg_dir')
    p.add_argument('--h_neg_dir', type=str, default=None,
                   help='--h_directions: images without the attribute, the first --n_train_img of them by name')
    p.add_argument('--h_direction_out', type=str, default=None, help='--h_directions: output directory')
    p.add_argument('--h_direction', type=str, default=None,
                   help='--run_test: edit with this direction file of --h_directions instead of a Δh checkpoint: '
                        'h2 = hs_coeff_origin_h * h + α * d_t at every edit step, α = --hs_coeff_delta_h as given '
                        '(not scaled by n_train_step / n_test_step: a direction has no training grid); with '
                        '--delta_interpolation the rows are (1, v * α)')
    p.add_argument('--edit_region', type=str, default=None,
                   help='--run_test: edit only these face-parsing classes ("hair hat"; names of the 19 BiSeNet '
                        'labels, background skin l_brow r_brow l_eye r_eye eye_g l_ear r_ear ear_r nose mouth u_lip '
                        'l_lip neck neck_l cloth hair hat).  The origin pass is parsed with --seg_weights into one '
                        'mask per image, and every edit step ends blended into the origin pass outside it; the masks '
                        'are written next to the PNG as <file>_ngen<n>_region_mask.png')
    p.add_argument('--edit_region_dilate', type=int, default=0,
                   help='--edit_region: grow the mask by a (2r + 1)^2 square max filter, r in 0..32 pixels')
    p.add_argument('--edit_region_feather', type=float, default=0.0,
                   help='--edit_region: soften the mask edge with a Gaussian of this sigma in pixels, 0..16 (0: hard '
                        'edge)')
    p.add_argument('--region_compose', type=str, default=None,
                   help='--run_test: compose several attribute edits into one image, each in its own face-parsing '
                        'region ("smiling=mouth,u_lip,l_lip grey_hair=hair"; at most 8 attributes, no class shared).  '
                        'Each attribute runs with its own DeltaBlock (the checkpoint name\'s "attribute" replaced), '
                        't_edit and t_addnoise, as --attr_sweep; after every step its rows are replaced by a per-pixel '
                        'mix of the attributes and the origin pass, weighted by the --seg_weights masks of the origin '
                        'pass (--edit_region_dilate / --edit_region_feather apply to every mask, overlaps are '
                        'normalised).  The masks are written as <file>_ngen<n>_region_compose.png')
    p.add_argument('--exact_inversion', **sa,
                   help='--run_test: edit real images without inversion drift.  Each batch\'s input images are '
                        'inverted with DDIM (the cached x_T is not used) and every edit step is anchored to that '
                        'inversion, so that an unedited pass returns the input image exactly and the origin row is '
                        'the input.  --edit_region / --region_compose parse the input image.  Needs --n_test_step '
                        '== --n_inv_step and DDIM sampling; the stochastic steps of --user_defined_t_addnoise draw '
                        'no noise')
    return p


def parse_args_and_config(argv=None):
    args = build_parser().parse_args(argv)
    config = load_config(args.config)
    args.exp = args.exp + f'_LC_{config.data.category}_t{args.t_0}_ninv{args.n_inv_step}_ngen{args.n_train_step}'
    level = getattr(logging, args.verbose.upper(), None)
    if not isinstance(level, int):
        raise ValueError('level {} not supported'.format(args.verbose))
    logging.basicConfig(level=level, format='%(levelname)s - %(filename)s - %(asctime)s - %(message)s')
    for d in ('checkpoint', 'checkpoint_latent', 'precomputed', 'runs', args.exp):
        os.makedirs(d, exist_ok=True)
    args.test_image_folder = os.path.join(args.exp, 'test_images', str(args.n_test_step))
    args.image_folder = os.path.join(args.exp, 'image_samples')
    os.makedirs(args.test_image_folder, exist_ok=True)
    os.makedirs(args.image_folder, exist_ok=True)
    torch.manual_seed(args.seed)
    np.random.seed(args.seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(args.seed)
    return args, config


def main(argv=None):
    args, config = parse_args_and_config(argv)
    from .diffusion_latent import Asyrp
    for flag in ("lpips", "h_directions"):
        if getattr(args, flag) and int(os.environ.get("WORLD_SIZE", "1")) > 1:
            logging.error(f"--{flag} computes statistics over every image: run it single-process, not under torchrun")
            return 1
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    runner = Asyrp(args, config)
    try:
        if args.diff_style:
            runner.run_diff_style()
        elif args.h_directions:
            runner.run_h_directions()
        elif args.run_test:
            runner.run_test()
        elif args.lpips:
            runner.compute_lpips_distance()
        else:
            print('Choose one mode! (this build implements --run_test, --lpips, --diff_style and --h_directions)')
            raise ValueError
    except Exception:
        logging.error(traceback.format_exc())
        return 1
    return 0


if __name__ == '__main__':
    sys.exit(main())
