"""fp32 functional restatement of U^2-Net (U-2-Net `model/u2net.py`; graph in hi3d_official_b200/u2net.py), seeded weights for
the full (U2NET) and `p` (U2NETP) widths, and the literal host steps of rembg 2.0.57's `remove` (bg.py, sessions/u2net.py) for
the default u2net session with the network passed in."""
import numpy as np
import torch
import torch.nn.functional as F

# The graph table, stated here from U-2-Net's model/u2net.py rather than taken from the module under test: the RSU depth of each
# stage, whether it pools (RSU-L) or not (RSU4F: stages 5, 6 and 5d), and the dilation of every REBNCONV.
STAGE_KIND = dict(stage1=(7, True), stage2=(6, True), stage3=(5, True), stage4=(4, True), stage5=(4, False), stage6=(4, False),
                  stage5d=(4, False), stage4d=(4, True), stage3d=(5, True), stage2d=(6, True), stage1d=(7, True))
DILATIONS = {
    (7, True): dict(rebnconvin=1, rebnconv1=1, rebnconv2=1, rebnconv3=1, rebnconv4=1, rebnconv5=1, rebnconv6=1, rebnconv7=2,
                    rebnconv6d=1, rebnconv5d=1, rebnconv4d=1, rebnconv3d=1, rebnconv2d=1, rebnconv1d=1),
    (6, True): dict(rebnconvin=1, rebnconv1=1, rebnconv2=1, rebnconv3=1, rebnconv4=1, rebnconv5=1, rebnconv6=2,
                    rebnconv5d=1, rebnconv4d=1, rebnconv3d=1, rebnconv2d=1, rebnconv1d=1),
    (5, True): dict(rebnconvin=1, rebnconv1=1, rebnconv2=1, rebnconv3=1, rebnconv4=1, rebnconv5=2,
                    rebnconv4d=1, rebnconv3d=1, rebnconv2d=1, rebnconv1d=1),
    (4, True): dict(rebnconvin=1, rebnconv1=1, rebnconv2=1, rebnconv3=1, rebnconv4=2, rebnconv3d=1, rebnconv2d=1, rebnconv1d=1),
    (4, False): dict(rebnconvin=1, rebnconv1=1, rebnconv2=2, rebnconv3=4, rebnconv4=8, rebnconv3d=4, rebnconv2d=2, rebnconv1d=1),
}

FULL = dict(stage1=(3, 32, 64), stage2=(64, 32, 128), stage3=(128, 64, 256), stage4=(256, 128, 512), stage5=(512, 256, 512),
            stage6=(512, 256, 512), stage5d=(1024, 256, 512), stage4d=(1024, 128, 256), stage3d=(512, 64, 128),
            stage2d=(256, 32, 64), stage1d=(128, 16, 64))
SMALL = dict(stage1=(3, 16, 64), stage2=(64, 16, 64), stage3=(64, 16, 64), stage4=(64, 16, 64), stage5=(64, 16, 64),
             stage6=(64, 16, 64), stage5d=(128, 16, 64), stage4d=(128, 16, 64), stage3d=(128, 16, 64), stage2d=(128, 16, 64),
             stage1d=(128, 16, 64))
VARIANTS = {"full": FULL, "p": SMALL}
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def up(a, b):
    return F.interpolate(a, size=b.shape[2:], mode="bilinear", align_corners=False)


def pool(x):
    return F.max_pool2d(x, 2, 2, ceil_mode=True)


def rebnconv(sd, p, x, d):
    y = F.conv2d(x, sd[p + "conv_s1.weight"], sd[p + "conv_s1.bias"], padding=d, dilation=d)
    y = F.batch_norm(y, sd[p + "bn_s1.running_mean"], sd[p + "bn_s1.running_var"], sd[p + "bn_s1.weight"], sd[p + "bn_s1.bias"],
                     False, 0.0, 1e-5)
    return F.relu(y)


def rsu(conv, stage, x):
    """conv(name, x, dilation) -> relu(BN(conv)); the RSU-L / RSU4F graph of u2net.py."""
    L, pooled = STAGE_KIND[stage]
    dil = DILATIONS[(L, pooled)]
    c = lambda name, t: conv(f"{stage}.{name}", t, dil[name])   # noqa: E731
    hxin = c("rebnconvin", x)
    hx = [None, c("rebnconv1", hxin)]
    for k in range(2, L):
        hx.append(c(f"rebnconv{k}", pool(hx[-1]) if pooled else hx[-1]))
    d = c(f"rebnconv{L - 1}d", torch.cat([c(f"rebnconv{L}", hx[L - 1]), hx[L - 1]], 1))
    for k in range(L - 2, 0, -1):
        d = c(f"rebnconv{k}d", torch.cat([up(d, hx[k]) if pooled else d, hx[k]], 1))
    return d + hxin


def u2net_graph(conv, x):
    """Encoder / decoder stages; returns the six stage outputs the side heads read: hx1d .. hx5d, hx6."""
    enc = []
    h = x
    for k in range(1, 7):
        h = rsu(conv, f"stage{k}", pool(h) if k > 1 else h)
        enc.append(h)
    d, dec = enc[5], [None] * 5
    for k in range(5, 0, -1):
        d = rsu(conv, f"stage{k}d", torch.cat([up(d, enc[k - 1]), enc[k - 1]], 1))
        dec[k - 1] = d
    return dec + [enc[5]]


def u2net_d0(sd, x):
    """d0 (before the sigmoid) of U2NET.forward with eval BatchNorm."""
    hs = u2net_graph(lambda name, t, d: rebnconv(sd, name + ".", t, d), x)
    ds = [F.conv2d(h, sd[f"side{k + 1}.weight"], sd[f"side{k + 1}.bias"], padding=1) for k, h in enumerate(hs)]
    ds = [ds[0]] + [up(t, ds[0]) for t in ds[1:]]
    return F.conv2d(torch.cat(ds, 1), sd["outconv.weight"], sd["outconv.bias"])[:, 0]


def u2net_forward(sd, x):
    """Output 0 of U2NET.forward: sigmoid(d0), (n, H, W)."""
    return torch.sigmoid(u2net_d0(sd, x))


def folded_d0(fold, x):
    """d0 from hi3d_official_b200.u2net.fold's tensors: BatchNorm inside the convs, outconv inside the side heads."""
    def conv(name, t, d):
        w, b, _ = fold[name]
        return F.relu(F.conv2d(t, w.to(t), b.to(t), padding=d, dilation=d))
    hs = u2net_graph(conv, x)
    out = fold["b0"]
    for (w, b), h in zip(fold["sides"], hs):
        out = out + up(F.conv2d(h, w.to(h), b.to(h), padding=1), x)
    return out[:, 0]


def random_u2net_sd(seed=0, variant="full", calib_hw=320):
    """Seeded U^2-Net state dict of the given widths, as U-2-Net's nn.Module would save it (num_batches_tracked included).
    He-initialised convs; each BatchNorm's running statistics are the batch statistics of its conv on a random calibration image
    of calib_hw^2 (the size the tower runs at: the dilated convs of the small deep levels see mostly padding, so statistics taken
    at another size do not transfer) and its affine is mildly random, so activations stay O(1) through all 119 convs.  The side
    heads and outconv give d0 a spread of several units per image, so that the min-max normalised mask is not noise."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)   # noqa: E731
    ur = lambda lo, hi, *s: lo + (hi - lo) * torch.rand(*s, generator=g)   # noqa: E731
    widths = VARIANTS[variant]
    sd = {}
    for stage, (cin, mid, cout) in widths.items():
        L, pooled = STAGE_KIND[stage]
        names = list(DILATIONS[(L, pooled)])
        for name in names:
            if name == "rebnconvin":
                ci, co = cin, cout
            elif name == "rebnconv1d":
                ci, co = 2 * mid, cout
            elif name == "rebnconv1":
                ci, co = cout, mid
            elif name.endswith("d"):
                ci, co = 2 * mid, mid
            else:
                ci, co = mid, mid
            p = f"{stage}.{name}."
            sd[p + "conv_s1.weight"] = rn(co, ci, 3, 3) * (2.0 / (9 * ci)) ** 0.5
            sd[p + "conv_s1.bias"] = rn(co) * 0.1
            sd[p + "bn_s1.weight"] = ur(0.3, 0.6, co)
            sd[p + "bn_s1.bias"] = 0.3 + rn(co) * 0.2
            sd[p + "bn_s1.running_mean"] = torch.zeros(co)
            sd[p + "bn_s1.running_var"] = torch.ones(co)
            sd[p + "bn_s1.num_batches_tracked"] = torch.tensor(0)
    side_in = [widths[f"stage{k}d"][2] for k in range(1, 6)] + [widths["stage6"][2]]
    for k, ci in enumerate(side_in, 1):
        sd[f"side{k}.weight"] = rn(1, ci, 3, 3) * (3.0 / (9 * ci)) ** 0.5
        sd[f"side{k}.bias"] = rn(1) * 0.1
    sd["outconv.weight"] = ur(1.0, 2.0, 1, 6, 1, 1)
    sd["outconv.bias"] = rn(1) * 0.1

    # calibration: running statistics = batch statistics of each conv's output (conv order = forward order)
    def calib_conv(name, t, d):
        p = name + "."
        y = F.conv2d(t, sd[p + "conv_s1.weight"], sd[p + "conv_s1.bias"], padding=d, dilation=d)
        sd[p + "bn_s1.running_mean"] = y.mean(dim=(0, 2, 3))
        v = y.var(dim=(0, 2, 3), unbiased=False)
        sd[p + "bn_s1.running_var"] = v.clamp_min(0.25 * float(v.mean()) + 1e-4)      # no near-constant channel is amplified
        return rebnconv(sd, p, t, d)
    with torch.no_grad():
        u2net_graph(calib_conv, rn(1, 3, calib_hw, calib_hw))
    return sd


def relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


# ---- rembg 2.0.57, remove(img, session=new_session()) with the u2net session, restated literally -------------------------------------
def rembg_normalize(img):
    """sessions/base.py normalize at (320, 320): RGB, LANCZOS, / max, ImageNet mean / std -> float32 (1, 3, 320, 320)."""
    from PIL import Image
    im = img.convert("RGB").resize((320, 320), Image.LANCZOS)
    im_ary = np.array(im)
    im_ary = im_ary / np.max(im_ary)
    tmp = np.zeros((im_ary.shape[0], im_ary.shape[1], 3))
    for c in range(3):
        tmp[:, :, c] = (im_ary[:, :, c] - MEAN[c]) / STD[c]
    return np.expand_dims(tmp.transpose((2, 0, 1)), 0).astype(np.float32)


def rembg_remove(img, net):
    """bg.remove -> fix_image_orientation, U2netSession.predict, naive_cutout; `net`: float32 (1, 3, 320, 320) array ->
    (1, 320, 320) probability (any array-like)."""
    from PIL import Image, ImageOps
    img = ImageOps.exif_transpose(img)
    pred = np.asarray(net(rembg_normalize(img)), dtype=np.float32)[0]
    ma, mi = np.max(pred), np.min(pred)
    pred = (pred - mi) / (ma - mi)
    mask = Image.fromarray((pred * 255).astype("uint8"), mode="L").resize(img.size, Image.LANCZOS)
    empty = Image.new("RGBA", img.size, 0)
    return Image.composite(img, empty, mask)
