"""fp64 reference of ops.token_logprobs: the log-softmax of the bf16 logits in float64, and the top n by a stable sort on
(-value, id), so ties go to the lowest id.  Entries past V hold id -1 and logprob -inf."""
import torch


def token_logprobs_ref(logits: torch.Tensor, tokens: torch.Tensor, n: int):
    """logits [R, V] (any float dtype, read as given), tokens int64 [R] -> (lp [R] f64, top_ids [R, n] int64, top_lp [R, n] f64)."""
    x = logits.detach().to("cpu", torch.float64)
    R, V = x.shape
    lsm = torch.log_softmax(x, dim=-1)
    lp = lsm.gather(1, tokens.to("cpu", torch.int64).view(R, 1)).view(R)
    ids = torch.full((R, n), -1, dtype=torch.int64)
    top = torch.full((R, n), float("-inf"), dtype=torch.float64)
    m = min(n, V)
    if m:
        order = torch.sort(-x, dim=-1, stable=True).indices[:, :m]   # value desc; a stable sort keeps ties in id order
        ids[:, :m] = order
        top[:, :m] = lsm.gather(1, order)
    return lp, ids, top


def lp_bound(lp64: torch.Tensor) -> torch.Tensor:
    """The bar an fp32 kernel is held to: 3e-5 + 1e-6 |lp64|."""
    return 3e-5 + 1e-6 * lp64.abs()
