"""Generate tests/golden/arcface_irse50.npz by running the REFERENCE'S OWN ArcFace Backbone(112, 50, 'ir_se') and
IDLoss (imported from /root/reference, which only exists in the build container, the way make_golden.py imports it) on
the seeded weights of asyrp_official_b200.synthetic.arcface_state_dict.

    python tests/golden/make_arcface_golden.py

IDLoss.__init__ reads pretrained/model_ir_se50.pth from disk, so the instance is built without it (IDLoss.__new__ +
nn.Module.__init__) and given the seeded facenet and the face_pool __init__ would make; extract_feats and forward are
the reference's own.  The fixture holds no weights: the seed and a SHA-256 of the drawn tensors pin them.

    seed, weights_sha256   synthetic.arcface_state_dict(seed), hashed by arcface_weights_sha256
    x_u8, x_hat_u8         [2][3][224][224] uint8 seeded smooth images (x_hat: x plus a smooth edit); the networks see
                           to_float(u8) = u8 / 127.5 - 1 in fp32, as an 8-bit image file would give them, which keeps
                           the fixture small
    pooled                 the 112 x 112 input of the backbone for x (the crop and AdaptiveAvgPool2d)
    feats, feats_hat       IDLoss.extract_feats of x and x_hat, [2][512]
    id_loss                IDLoss.forward(x, x_hat), [2]
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from asyrp_official_b200 import synthetic  # noqa: E402

from losses.id_loss import IDLoss  # noqa: E402  (reference)
from models.insight_face.model_irse import Backbone  # noqa: E402  (reference)

SEED = 7
SIZE = 224


def arcface_weights_sha256(sd):
    """SHA-256 over the sorted keys and the fp32 bytes of every floating tensor"""
    h = hashlib.sha256()
    for k in sorted(sd):
        if sd[k].is_floating_point():
            h.update(k.encode())
            h.update(sd[k].float().contiguous().numpy().tobytes())
    return h.hexdigest()


def images(seed):
    """sums of a few low-frequency sinusoids per channel, fp32 in [-1, 1]"""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, SIZE), torch.linspace(0, 1, SIZE), indexing="ij")
    out = torch.zeros(2, 3, SIZE, SIZE)
    for _ in range(4):
        fy, fx, ph = (torch.rand(2, 3, 1, 1, generator=g) * 8 for _ in range(3))
        out += torch.sin(fy * yy * 3.14 + fx * xx * 3.14 + ph)
    return (out / 4).clamp(-1, 1)


def to_u8(x):
    return torch.round((x + 1) * 127.5).clamp(0, 255).to(torch.uint8)


def to_float(u8):
    """the fp32 image of a uint8 one, as the fixture's readers compute it"""
    return torch.as_tensor(u8).float() / 127.5 - 1


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    sd = synthetic.arcface_state_dict(seed=SEED)
    facenet = Backbone(input_size=112, num_layers=50, drop_ratio=0.6, mode='ir_se')
    facenet.load_state_dict(sd, strict=True)
    facenet.eval()
    loss = IDLoss.__new__(IDLoss)
    torch.nn.Module.__init__(loss)
    loss.facenet = facenet
    loss.face_pool = torch.nn.AdaptiveAvgPool2d((112, 112))
    x_u8 = to_u8(images(1))
    x_hat_u8 = to_u8((images(1) + 0.2 * images(2)).clamp(-1, 1))
    x, x_hat = to_float(x_u8), to_float(x_hat_u8)
    with torch.no_grad():
        pooled = loss.face_pool(x[:, :, 35:223, 32:220])
        feats = loss.extract_feats(x)
        feats_hat = loss.extract_feats(x_hat)
        id_loss = loss(x, x_hat)
    n_params = sum(v.numel() for k, v in facenet.state_dict().items() if not k.endswith("num_batches_tracked"))
    print(f"Backbone(112, 50, 'ir_se'): {len(facenet.state_dict())} keys, {n_params / 1e6:.1f} M parameters; "
          f"IDLoss {id_loss.tolist()}")
    np.savez_compressed(os.path.join(HERE, "arcface_irse50.npz"), seed=np.int64(SEED),
                        weights_sha256=np.array(arcface_weights_sha256(sd)), x_u8=x_u8.numpy(),
                        x_hat_u8=x_hat_u8.numpy(),
                        pooled=pooled.numpy(), feats=feats.numpy(), feats_hat=feats_hat.numpy(),
                        id_loss=id_loss.numpy())


if __name__ == "__main__":
    main()
