"""fp64 restatement of per-image exposure compensation (DESIGN.md §6k, csrc/exposure.cu).

Exposures e [n_img, 3] in stops, gains g = 2^e.  Rows are visited through rays_a [n, 3] = (ray, start, count); each
ray's image is img[ray], clamped to [0, n_img) as the kernels clamp it."""
import numpy as np

LN2 = np.log(2.0)


def _rays(rays_a, n_rows):
    for ray, start, cnt in np.asarray(rays_a, np.int64):
        cnt = min(cnt, n_rows - start)
        if cnt > 0 and start >= 0:
            yield ray, start, cnt


def _image(img, ray, n_img):
    img = np.asarray(img, np.int64).reshape(-1)
    i = img[0] if img.size == 1 else img[ray]
    return int(min(max(i, 0), n_img - 1))


def apply(rgbs, rays_a, img, expo):
    """c' = 2^e[img(ray)] c over every ray's rows, fp64; rows outside every ray are NaN."""
    c = np.asarray(rgbs, np.float64)
    e = np.asarray(expo, np.float64)[:, :3]
    out = np.full_like(c, np.nan)
    for ray, s, k in _rays(rays_a, len(c)):
        out[s:s + k] = np.exp2(e[_image(img, ray, len(e))]) * c[s:s + k]
    return out


def bwd(out, drgbs, rays_a, img, expo):
    """(dL/dc = g dL/dc' per row, grad [n_img, 3] = ln2 sum dL/dc' c' per image, sum |term| per image), fp64."""
    o, d = np.asarray(out, np.float64), np.asarray(drgbs, np.float64)
    e = np.asarray(expo, np.float64)[:, :3]
    dc = d.copy()
    grad, mag = np.zeros_like(e), np.zeros_like(e)
    for ray, s, k in _rays(rays_a, len(d)):
        i = _image(img, ray, len(e))
        dc[s:s + k] = np.exp2(e[i]) * d[s:s + k]
        t = LN2 * d[s:s + k] * o[s:s + k]
        grad[i] += t.sum(0)
        mag[i] += np.abs(t).sum(0)
    return dc, grad, mag


def adam(e, g, m, v, hyper, lr_ratio, beta1=0.9, beta2=0.999, eps=1e-15, found_inf=False, project=True):
    """One exposure Adam step: hyper = (lr / bc1, sqrt(bc2), inv_scale); gg = g inv_scale, m, v as torch's Adam,
    e -= lr_ratio lr/bc1 m / (sqrt(v) / sqrt(bc2) + eps), then e -= mean_i e per channel.  found_inf: nothing but the
    gradient changes; project=False leaves out the projection.  Returns (e, g = 0, m, v) in fp64."""
    e, g, m, v = (np.array(x, np.float64) for x in (e, g, m, v))
    if found_inf:
        return e, np.zeros_like(g), m, v
    lr_bc1, bc2, inv = (float(x) for x in hyper[:3])
    gg = g * inv
    m = m + (gg - m) * (1 - beta1)
    v = v * beta2 + (1 - beta2) * gg * gg
    e = e - lr_ratio * lr_bc1 * m / (np.sqrt(v) / bc2 + eps)
    return (e - e.mean(0)) if project else e, np.zeros_like(g), m, v
