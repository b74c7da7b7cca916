"""Reference and error bound for hqq_b200_lm_logprob (include/hqq_b200.h states the numbers it computes).

The float64 reference takes the T-rounded float64 logits L[m][v] = T(sum_k x[m][k] W[v][k]) and returns lse[m] = log sum_v exp(L[m][v])
and tgt[m] = L[m][target] (-inf outside the shard).  The kernel differs from it in three places, and the bound adds them up:
  1. each logit: fp32 accumulation over K products (at most gamma_K * sum_k |x_k W_vk|, gamma_K = K u32 / (1 - K u32)) before the
     one rounding to T, so the two T-rounded logits differ by at most that plus one ulp of T at the logit's magnitude;
  2. lse is 1-Lipschitz in the max norm of the logits (its gradient is a probability vector): the largest logit error carries over;
  3. fp32 arithmetic of the reduction: every term of S passes through three expf (<= 2 ulp each), three fp32 subtractions inside
     their arguments (l - m_w, m_w - m_j, m_j - M; error <= u32 |argument| <= 2 u32 max |L| each), two products and at most
     n_tiles + 12 additions; logf (<= 1 ulp) and the final add cost u32 |lse| each.
tgt only carries 1.
`model()` restates the kernel's reduction in float32 (warp partials, warp merge, tile merge) with four plantable defects."""
import math

import torch

U32 = 2.0 ** -24
TILE = 128


def ulp(t_dtype, mag):
    """One ulp of T at magnitude `mag` (a float64 tensor), subnormals included."""
    bits = 10 if t_dtype == torch.float16 else 7
    emin = -14 if t_dtype == torch.float16 else -126
    e = torch.floor(torch.log2(mag.clamp_min(2.0 ** emin)))
    return torch.pow(2.0, e - bits)


def reference(x, W, targets, index_offset):
    """float64 lse and tgt of the T-rounded float64 logits; also returns the logits and sum_k |x W| (the accumulation bound's scale)."""
    xd, Wd = x.double(), W.double()
    d = xd @ Wd.t()
    L = d.to(x.dtype).double()
    lse = torch.logsumexp(L, dim=1)
    N = W.shape[0]
    t = targets - index_offset
    inside = (t >= 0) & (t < N)
    tgt = torch.full_like(lse, -math.inf)
    rows = torch.nonzero(inside).flatten()
    tgt[rows] = L[rows, t[rows]]
    absdot = xd.abs() @ Wd.abs().t()
    return lse, tgt, L, absdot


def bounds(x, W, targets, index_offset, L, absdot, lse):
    """Per-position bounds on |lse - ref| and |tgt - ref| (see the module docstring)."""
    K, N = x.shape[1], W.shape[0]
    gamma = K * U32 / (1 - K * U32)
    acc = gamma * absdot                                   # [M, N]
    dlogit = acc + ulp(x.dtype, L.abs() + acc)             # per logit
    n_tiles = -(-N // TILE)
    maxabs = L.abs().max(dim=1).values
    # relative error of S: three expf (2 ulp = 4 u each at worst), two products, n_tiles + 12 additions, three argument subtractions
    rel_s = (2 * (n_tiles + 20) + 6 * 2 * maxabs) * U32 * 1.01
    b_lse = dlogit.max(dim=1).values + rel_s + 3 * U32 * (lse.abs() + maxabs + math.log(N) + 1)  # + logf and the final add
    t = targets - index_offset
    inside = (t >= 0) & (t < N)
    b_tgt = torch.zeros_like(b_lse)
    rows = torch.nonzero(inside).flatten()
    b_tgt[rows] = dlogit[rows, t[rows]]
    return b_lse, b_tgt


def model(L, targets, index_offset, defect=None):
    """The kernel's reduction in float32 over the T-rounded logits L [M, N] (float64 holding T values).  defect: "target_off_by_one",
    "drop_tile" (vocabulary tile 1, or 0 when there is one), "no_mask" (rows past N count as logit 0) or "no_rescale" (tile partials
    summed without exp(m_j - M))."""
    M, N = L.shape
    n_tiles = -(-N // TILE)
    Lf = torch.full((M, n_tiles * TILE), 0.0 if defect == "no_mask" else -math.inf, dtype=torch.float32)
    Lf[:, :N] = L.float()
    tl = Lf.view(M, n_tiles, 8, 16)                        # [M, tile, warp, 16 rows]
    mw = tl.max(dim=3).values                              # warp maxima
    sw = torch.where(mw.isinf(), torch.zeros_like(mw), torch.exp(tl - mw.unsqueeze(3)).sum(dim=3))
    mj = mw.max(dim=2).values                              # tile maxima
    sj = (sw * torch.exp(mw - mj.unsqueeze(2))).sum(dim=2)
    keep = torch.ones(n_tiles, dtype=torch.bool)
    if defect == "drop_tile":
        keep[1 if n_tiles > 1 else 0] = False
    mj, sj = mj[:, keep], sj[:, keep]
    Mx = mj.max(dim=1).values
    S = sj.sum(dim=1) if defect == "no_rescale" else (sj * torch.exp(mj - Mx.unsqueeze(1))).sum(dim=1)
    lse = (Mx + torch.log(S)).double()
    t = targets - index_offset + (1 if defect == "target_off_by_one" else 0)
    inside = (t >= 0) & (t < N)
    tgt = torch.full((M,), -math.inf, dtype=torch.float64)
    rows = torch.nonzero(inside).flatten()
    tgt[rows] = L[rows, t[rows]]
    return lse, tgt
