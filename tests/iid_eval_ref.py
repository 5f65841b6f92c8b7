"""The intrinsic-image evaluation step restated for the IID evaluation tests: compute_iid_metric (src/util/metric.py:
263-338) for PSNR and SSIM as script/iid/eval.py:182-213 calls it, with the colour transforms of image_util.py:144-149.
torchmetrics is not a dependency, so PeakSignalNoiseRatio and StructuralSimilarityIndexMeasure (data_range=1.0) are
restated from their definitions (torchmetrics/functional/image/psnr.py and ssim.py).

Two variants of one code path, on the device the inputs are on:
- float32: what the reference computes (torch.linalg.lstsq, torch.quantile, float32 metric arithmetic);
- float64: the bound reference (the scale as sum pg / sum p^2, every step in float64)."""
import numpy as np
import torch
import torch.nn.functional as F

UP_TO_SCALE = ("shading", "residual")
TRANSFORMS = (None, "srgb2linear", "linear2srgb")


def colour(x: torch.Tensor, transform):
    if transform == "srgb2linear":
        return x ** 2.2
    if transform == "linear2srgb":
        return x ** (1.0 / 2.2)
    assert transform is None, transform
    return x


def psnr(pred: torch.Tensor, gt: torch.Tensor) -> torch.Tensor:
    """PeakSignalNoiseRatio(data_range=1.0): (2 ln(range) - ln(SSE / n)) * 10 / ln(10), in the inputs' dtype."""
    sse = torch.sum(torch.pow(pred - gt, 2))
    one = torch.tensor(1.0, dtype=pred.dtype, device=pred.device)
    return (2 * torch.log(one) - torch.log(sse / pred.numel())) * (10 / torch.log(torch.tensor(10.0, dtype=pred.dtype)))


def gaussian(dtype, device) -> torch.Tensor:
    """torchmetrics' _gaussian(11, 1.5): exp(-(d / 1.5)^2 / 2) over d = -5..5, normalised."""
    d = torch.arange(-5, 6, 1, dtype=dtype, device=device)
    g = torch.exp(-torch.pow(d / 1.5, 2) / 2)
    return g / g.sum()


def ssim(pred: torch.Tensor, gt: torch.Tensor) -> torch.Tensor:
    """StructuralSimilarityIndexMeasure(data_range=1.0) of [1, 3, H, W] maps: Gaussian window (sigma 1.5, 11 x 11, the
    outer product of the 1-D weights), reflect padding of 5, crop of 5, mean of the SSIM map."""
    g = gaussian(pred.dtype, pred.device)
    kernel = torch.matmul(g[:, None], g[None, :]).expand(3, 1, 11, 11)
    c1, c2 = (0.01 * 1.0) ** 2, (0.03 * 1.0) ** 2
    p = F.pad(pred, (5, 5, 5, 5), mode="reflect")
    t = F.pad(gt, (5, 5, 5, 5), mode="reflect")
    mu_p, mu_t, e_pp, e_tt, e_pt = F.conv2d(torch.cat((p, t, p * p, t * t, p * t)), kernel, groups=3).split(1)
    mu_pp, mu_tt, mu_pt = mu_p.pow(2), mu_t.pow(2), mu_p * mu_t
    s_pp = torch.clamp(e_pp - mu_pp, min=0.0)
    s_tt = torch.clamp(e_tt - mu_tt, min=0.0)
    s_pt = e_pt - mu_pt
    upper = 2 * s_pt + c2
    lower = s_pp + s_tt + c2
    full = ((2 * mu_pt + c1) * upper) / ((mu_pp + mu_tt + c1) * lower)
    return full[..., 5:-5, 5:-5].reshape(1, -1).mean(-1).mean()


def brightness(gt: torch.Tensor) -> torch.Tensor:
    return 0.3 * gt[0] + 0.59 * gt[1] + 0.11 * gt[2]


def evaluate(pred, gt, target_name, mask=None, transform=None, dtype=torch.float32, scale=None):
    """One (sample, target) pair: ({"psnr", "ssim"}, {"n_valid", "scale", "quantile", "quantile_scale", "pred", "gt"}),
    where pred / gt are the [3, H, W] maps the metrics see (before the SSIM zeroing). pred, gt [3, H, W]; mask bool
    [3, H, W] or None. Raises (torch.quantile) for an up-to-scale target without a pixel valid in mask channel 0.
    scale: use this least-squares scale instead of fitting it. torch's CPU lstsq returns slightly different float32
    values for the same inputs from one call to the next, so a fixture's scale is pinned this way."""
    pred, gt = colour(pred.to(dtype), transform), colour(gt.to(dtype), transform)
    info = {"scale": None, "quantile": None, "quantile_scale": None}
    if target_name in UP_TO_SCALE:
        m = mask if mask is not None else torch.ones(pred.shape, dtype=torch.bool, device=pred.device)
        p, g = pred[m].reshape(-1, 1), gt[m].reshape(-1, 1)
        if scale is not None:
            s = torch.tensor([[scale]], dtype=dtype, device=pred.device)
        elif dtype == torch.float32:
            s = torch.linalg.lstsq(p, g)[0]                                   # [1, 1]
        else:
            den = (p * p).sum()
            s = torch.where(den == 0, torch.zeros_like(den), (p * g).sum() / den)
        pred = s * pred
        q = torch.quantile(brightness(gt)[m[0]], 0.9)
        k = 0 if q < 1e-4 else float(0.8 / q)
        gt, pred = torch.clamp(k * gt, 0, 1), torch.clamp(k * pred, 0, 1)
        info.update(scale=float(s.reshape(-1)[0]), quantile=float(q), quantile_scale=float(k))
    info.update(pred=pred, gt=gt, n_valid=pred.numel() if mask is None else int(mask.sum()))
    if mask is None:
        out = {"psnr": psnr(pred, gt), "ssim": ssim(pred[None], gt[None])}
    else:
        z = torch.zeros((), dtype=dtype, device=pred.device)
        out = {"psnr": psnr(pred[mask], gt[mask]),
               "ssim": ssim(torch.where(mask, pred, z)[None], torch.where(mask, gt, z)[None])}
    return {k: float(v) for k, v in out.items()}, info


def quantile_order_statistics(gt, mask=None, transform=None):
    """(v[floor r], v[ceil r], w) of torch.quantile(brightness, 0.9) in float32: r = fl32(0.9f * (n - 1)), w = r - floor r,
    v the sorted brightness of the pixels valid in mask channel 0. Computed on the device the inputs are on."""
    b = brightness(colour(gt.float(), transform))
    b = (b[mask[0]] if mask is not None else b.reshape(-1)).sort().values.cpu().numpy()
    r = np.float32(0.9) * np.float32(b.size - 1)
    lo, hi = int(np.floor(r)), int(np.ceil(r))
    return b[lo], b[hi], np.float32(r - np.float32(lo))


def lerp_f32(a, b, w):
    """torch's lerp (Lerp.h) in float32 without contraction."""
    a, b, w = np.float32(a), np.float32(b), np.float32(w)
    d = np.float32(b - a)
    return np.float32(a + np.float32(w * d)) if w < 0.5 else np.float32(b - np.float32(d * np.float32(1 - w)))
