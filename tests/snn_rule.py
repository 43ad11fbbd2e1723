"""Expected values of the SNN matcher (ag_match_snn / ag_match_pairs), shared by tests/test_match_pairs_cpu.py and
tests/test_gpu_match_pairs.py."""
import torch


def snn_expected(dist, ratio=0.8):
    """The matcher's rule spelled out with torch reductions on a distance matrix [n1,n2] (n1, n2 >= 1; any device), independently of the
    matcher's kernels: min by value with NaN ignored, idx2 = the first column equal to the min ((+inf, column 0) for a row with nothing
    below +inf), every idx2 column set to 100000, the NaN-ignoring minimum of that (+inf when nothing is left), keep = min / (second +
    1e-8) <= ratio in fp32.  -> (idx2 int64, min, second, keep bool, tent [ntent,2] int64 = (row, idx2[row]) of the kept rows)."""
    inf = torch.tensor(float("inf"), dtype=dist.dtype, device=dist.device)
    n1, n2 = dist.shape
    nan = torch.isnan(dist)
    mn = torch.where(nan, inf, dist).min(1).values
    cols = torch.arange(n2, device=dist.device).expand(n1, n2)
    first = torch.where((dist == mn[:, None]) & ~nan, cols, n2).min(1).values
    idx2 = torch.where(mn < inf, first, torch.zeros_like(first))
    mask = torch.zeros(n2, dtype=torch.bool, device=dist.device)
    mask[idx2] = True
    sec = torch.where(mask[None, :], torch.full_like(dist, 100000.0), dist)
    sec = torch.where(torch.isnan(sec), inf, sec).min(1).values
    keep = (mn / (sec + 1e-8)) <= ratio
    rows = torch.arange(n1, device=dist.device)
    return idx2, mn, sec, keep, torch.stack([rows[keep], idx2[keep]], 1)
