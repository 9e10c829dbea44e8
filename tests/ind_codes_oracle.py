"""float64 / numpy restatement of the per-image appearance codes of the stage-0 train path (include/n2m_b200_fused.h "Per-image
appearance codes"): the code columns the gather writes, the per-image code-gradient reduction and the two-group Adam step.

The reference (renderer.py:698-719, network.py:159-166, renderer.py:173-174): every sample of ray n sees individual_codes[index[n]]
appended to color_net's input, autocast rounds that input to fp16; the code gradient is the fp16 input gradient summed in fp32 per code
row (index backward); the codes are their own Adam group at 0.1 * lr, weight decay 0."""
import numpy as np

COL_CODE = 54
BETA1, BETA2 = 0.9, 0.999


def gather_code_cols(codes, ray_img, rec_ray, M, D, code_row=None):
    """tile columns 54..53+D of the first M rows: fp16(codes[ray_img[rec_ray[j]]]) (or fp16(code_row) for every row); [M, D] float64"""
    if code_row is not None:
        rows = np.broadcast_to(np.asarray(code_row, np.float32)[:D], (M, D))
    else:
        rows = np.asarray(codes, np.float32)[np.asarray(ray_img)[np.asarray(rec_ray[:M])], :D]
    return rows.astype(np.float16).astype(np.float64)


def part_rays(n, part, nparts):
    """rays [lo, hi) of ray-range part `part` of `nparts` of a batch of n rays (n2m_common.cuh part_first_ray: eighths of the batch)"""
    e0, e1 = part * 8 // nparts, (part + 1) * 8 // nparts
    return n * e0 // 8, n * e1 // 8


def code_grad(denc_codes, rays, ray_img, ind_num, D, M, n_active=None, part=0, nparts=1):
    """g[img, j] = sum over the samples s < M of every ray of the part of denc_codes[s, j] (the fp16 loss-scaled terms), float64.
    rays [N, 2] = (offset, count) of the march; n_active: the adaptive ray count (None: all N rays)."""
    rays = np.asarray(rays)
    N = rays.shape[0]
    n = N if n_active is None else min(max(int(n_active), 1), N)
    lo, hi = part_rays(n, part, nparts)
    g = np.zeros((ind_num, D))
    for r in range(lo, hi):
        off, cnt = int(rays[r, 0]), int(rays[r, 1])
        end = min(off + cnt, M)
        if end > off:
            g[int(ray_img[r])] += np.asarray(denc_codes[off:end, :D], np.float64).sum(0)
    return g


def adam_two_groups(ind, g_scaled, m, v, D, step, lr, loss_scale, found_inf, eps=1e-15):
    """one step of torch Adam (betas 0.9 / 0.999, no weight decay) on the block [64 D code columns at lr | codes at 0.1 lr] after
    GradScaler's unscale; skipped when found_inf.  Returns (ind, m, v) as new float64 arrays."""
    ind, m, v = (np.array(a, np.float64) for a in (ind, m, v))
    if found_inf:
        return ind, m, v
    g = np.asarray(g_scaled, np.float64) / loss_scale
    lrs = np.where(np.arange(ind.size) < 64 * D, lr, 0.1 * lr)
    m = BETA1 * m + (1 - BETA1) * g
    v = BETA2 * v + (1 - BETA2) * g * g
    bc1, bc2 = 1 - BETA1 ** step, 1 - BETA2 ** step
    ind = ind - lrs / bc1 * m / (np.sqrt(v) / np.sqrt(bc2) + eps)
    return ind, m, v
