"""2-GPU (NCCL) expert-parallel forward vs the single-device oracle.  Skipped unless >= 2 GPUs are visible (the
single-GPU run skips it; run on a machine with two GPUs: `python -m pytest tests/test_gpu_ep.py -m gpu`)."""
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

from ep_common import ep_worker, free_port

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
# NCCL all-to-all-v / NVLink peer-memory exchange (dispatch in the permute kernel, return in the fc2 epilogue)
@pytest.mark.parametrize("transport", ["cuda", "fused"])
@pytest.mark.parametrize("E,k,T,d,I", [(8, 2, 50, 256, 128), (64, 6, 1024, 2560, 1664)])
def test_ep_forward_two_gpus(E, k, T, d, I, transport):
    tc = dict(hidden_size=d, moe_num_experts=E, moe_topk=k, moe_intermediate_size=I, moe_num_shared_experts=2)
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(ep_worker, args=(2, free_port(), transport, "cuda", tc, T, "bfloat16", tmp), nprocs=2, join=True)
        for r in range(2):
            res = torch.load(f"{tmp}/rank{r}.pt")
            assert res["err_safe"] <= 1e-2 and res["n_safe"] >= res["n"] // 4, res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("E,k,T,d,I", [(8, 2, 60, 256, 128), (64, 6, 500, 256, 128)])
def test_ep_forward_backward_two_gpus(E, k, T, d, I):
    """BASELINE cfg 5 unit: expert-parallel MoE layer fwd+bwd, grads vs fp32 autograd through the oracle."""
    from ep_common import ep_train_worker
    tc = dict(hidden_size=d, moe_num_experts=E, moe_topk=k, moe_intermediate_size=I, moe_num_shared_experts=2)
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(ep_train_worker, args=(2, free_port(), tc, T, tmp), nprocs=2, join=True)
        for r in range(2):
            res = torch.load(f"{tmp}/rank{r}.pt")
            wtol = 2e-2 if res["all_safe"] else 1.5e-1
            assert res["out"] <= 1e-2 and res["dx"] <= 2e-2 and res["d_fc1"] <= wtol and res["d_fc2"] <= wtol, res

