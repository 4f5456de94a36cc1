"""float64 restatement of mipnerf_b200_interlevel_loss(_backward) (include/mipnerf_b200.h): mip-NeRF 360's interlevel
loss of proposal weights w_hat at fenceposts t_hat against fine weights w at fenceposts t, per ray, and its gradient
in w_hat.  The proposal range of each fine interval comes from exact fp32 comparisons, as in the kernel; the rest is
float64."""
import numpy as np

EPS = float(np.finfo(np.float32).eps)


def interlevel(t, w, t_hat, w_hat, chunk=64):
    """t [B,N+1], w [B,N], t_hat [B,M+1], w_hat [B,M] -> (loss [B], d loss / d w_hat [B,M], lo [B,N], hi [B,N])."""
    t, th = np.asarray(t, np.float32), np.asarray(t_hat, np.float32)
    w, wh = np.asarray(w, np.float64), np.asarray(w_hat, np.float64)
    B, N, M = w.shape[0], w.shape[1], wh.shape[1]
    loss, grad = np.zeros(B), np.zeros((B, M))
    lo, hi = np.zeros((B, N), np.int64), np.zeros((B, N), np.int64)
    for c0 in range(0, B, chunk):
        sl = slice(c0, min(B, c0 + chunk))
        le = (th[sl, None, :] <= t[sl, :-1, None]).sum(-1)
        lt = (th[sl, None, :] < t[sl, 1:, None]).sum(-1)
        lo[sl], hi[sl] = np.clip(le - 1, 0, M), np.clip(lt, 0, M)
        cdf = np.concatenate([np.zeros((wh[sl].shape[0], 1)), np.cumsum(wh[sl], axis=1)], axis=1)
        rows = np.arange(cdf.shape[0])[:, None]
        bound = np.where(hi[sl] > lo[sl], cdf[rows, hi[sl]] - cdf[rows, lo[sl]], 0.0)
        excess = np.maximum(0.0, w[sl] - bound)
        loss[sl] = (excess ** 2 / (w[sl] + EPS)).sum(axis=1)
        g = -2.0 * excess / (w[sl] + EPS)
        j = np.arange(M)
        cover = (j[None, None, :] >= lo[sl][..., None]) & (j[None, None, :] < hi[sl][..., None])  # [b, N, M]
        grad[sl] = (g[..., None] * cover).sum(axis=1)
    return loss, grad, lo, hi
