"""A torch restatement of the typical / epsilon / eta cuts as csrc/sampling.cu states them (sample_row<T, true>): set rules over the
probabilities, no sort.  K0 is what temperature / top-k / top-p kept; with s = the scaled logit and q = p / mass(K0), typical keeps
{|s - E_q[s]| <= d*}, d* the smallest deviation whose set holds typical_p of the mass; epsilon keeps p >= epsilon * mass(K1); eta keeps
p >= min(eta, sqrt(eta) * exp(-H(K2))) * mass(K2); epsilon and eta also keep the tokens tied at the largest logit of K1.  float64
throughout.  tests/golden/warpers_kats.npz pins it to transformers 5.5's warper chain."""
import torch


def base_keep(x: torch.Tensor, T: float, top_k: int, top_p: float) -> torch.Tensor:
    """HF's temperature, top-k and top-p over one fp32 row, in fp32 with HF's sort (so a tie split at the nucleus threshold is split
    as HF splits it): the kept mask."""
    s = x.float()[None] / T if T != 1.0 else x.float()[None]
    keep = torch.isfinite(s)
    if top_k != 0:
        keep &= s >= torch.topk(s, min(top_k, s.shape[-1]))[0][..., -1, None]
        s = torch.where(keep, s, -torch.inf)
    if top_p < 1.0:
        sv, si = torch.sort(s, descending=False)
        rm = sv.softmax(dim=-1).cumsum(dim=-1) <= (1 - top_p)
        rm[..., -1:] = False
        keep &= ~rm.scatter(1, si, rm)
    return keep[0]


def cuts(x: torch.Tensor, keep: torch.Tensor, T: float, typical_p: float, eps: float, eta: float, dev_slack: float = 0.0) -> torch.Tensor:
    """The typical / epsilon / eta cuts after ``keep`` (each on when HF turns it on) -> the final kept mask.  ``dev_slack`` moves
    typical's deviation threshold (the tolerance of the kernel's bisection)."""
    s = torch.where(keep, (x.float() / T if T != 1.0 else x.float()).double(), -torch.inf)  # HF's fp32 scores
    keep = keep.clone()
    if typical_p < 1.0:
        q = torch.softmax(s, 0)
        c = (q[keep] * s[keep]).sum()
        dev = torch.where(keep, (s - c).abs(), torch.inf)
        order = torch.argsort(dev)
        cum = torch.cumsum(q[order], 0)
        before = torch.cat([cum.new_zeros(1), cum])  # before[i]: the mass of the i closest tokens
        below = before[torch.searchsorted(dev[order], dev - dev_slack)]  # the mass strictly closer to c than each token (its tie group starts there)
        keep &= below < typical_p
    if 0.0 < eps < 1.0 or 0.0 < eta < 1.0:
        s = torch.where(keep, s, -torch.inf)
        top = s == s.max()
        if 0.0 < eps < 1.0:
            keep &= (torch.softmax(s, 0) >= eps) | top
            s = torch.where(keep, s, -torch.inf)
        if 0.0 < eta < 1.0:
            q = torch.softmax(s, 0)
            h = -(q[keep] * torch.log(q[keep])).sum()
            keep &= (q >= min(eta, eta ** 0.5 * float(torch.exp(-h)))) | top
    return keep


def kept(x, T, top_k, top_p, typical_p, eps, eta) -> torch.Tensor:
    return cuts(x, base_keep(x, T, top_k, top_p), T, typical_p, eps, eta)
