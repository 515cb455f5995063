"""Worker of tests/test_ep_tokens_multi_gpu.py (one process per GPU, torchrun): the expert-parallel MoE layer for any number of
tokens per rank on REAL peer memory, through the operator layer a user runs — a tiny DeepSeek-V3 model loaded with the H100 rule
file, its routed experts sharded over the ranks, `attach_expert_parallel`, then forward steps that each begin with
`PeerExchange.begin_step`.  The ranks run concurrently with no host synchronisation between steps: prompt chunks with different
token counts per rank (0, 1, 47, 48 and more), interleaved with decode steps of one token per rank (the one-launch kernel on the
same exchange).  Every rank's output must match the unsharded block (routed experts over all E, then the shared expert as a
second rounded term): same routing bits, output within fp32 re-association of the cross-rank sum."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from ktransformers_b200 import native  # noqa: E402

BF16 = 30


def bf16_close(a, b):
    a, b = a.float().cpu().numpy(), b.float().cpu().numpy()
    assert np.isfinite(a).all()
    ok = np.abs(a - b) <= 2 * 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()
    return bool(ok.all()) and float((a == b).mean()) >= 0.9, float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    from test_gpu_operators import _write_gguf, H, I, E, K
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.expert_parallel import attach_expert_parallel
    from ktransformers_b200.operators.experts import KExpertsB200
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    import ktransformers_b200.optimize.optimize as opt
    tmp = tempfile.mkdtemp(prefix=f"ep_tokens_{rank}_")
    _write_gguf(os.path.join(tmp, "tiny.gguf"))          # seeded: the same weights on every rank
    rule = os.path.join(os.path.dirname(opt.__file__), "optimize_rules", "DeepSeek-V3-Chat-b200.yaml")
    torch.set_default_dtype(torch.bfloat16)
    cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                           num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
    with torch.device("meta"):
        model = DeepseekV3MoEOnlyForCausalLM(cfg)
    optimize_and_load_gguf(model, rule, tmp, cfg, default_device="cuda")
    moe = model.model.layers[1].mlp
    full = moe.experts.generate_experts                  # the unsharded experts: the reference
    shard = KExpertsB200(full.key, full.gguf_loader, full.config, E, device="cuda", expert_parallel_rank=rank,
                         expert_parallel_size=world, hidden_dtype=torch.bfloat16)
    shard.load()
    moe.experts.generate_experts = shard
    ex = attach_expert_parallel(model, H, BF16, dev)

    # every rank draws the same schedule; token values differ per rank
    srng = np.random.default_rng(11)
    fixed = [0, 1, 47, 48, 5, 0, 30, 64][:world] + [0] * max(0, world - 8)
    steps = [fixed, [1] * world, [int(c) for c in srng.integers(0, 65, world)], [1] * world, [int(c) for c in srng.integers(0, 9, world)],
             [0] * world, list(reversed(fixed))]
    trng = torch.Generator(device="cpu").manual_seed(100 + rank)
    xs, outs = [], []
    for counts in steps:                                  # back to back: no device synchronisation between steps
        n = counts[rank]
        x = (torch.randn(1, n, H, generator=trng) / 10).to(torch.bfloat16).to(dev)
        assert ex.begin_step(n) == counts
        y = moe(x)
        xs.append(x)
        outs.append((y.clone(), *(t.clone() for t in moe.last_topk)) if n else (y.clone(), None, None))
    torch.cuda.synchronize()
    assert not ex.timed_out(), f"rank {rank}: a peer wait timed out"
    assert ex.step.counts is None, "the step counts expire after the step's MoE layers"

    lib, s = native.lib(), torch.cuda.current_stream().cuda_stream
    worst = 0.0
    for st, (counts, x, (y, idx, wt)) in enumerate(zip(steps, xs, outs)):
        n = counts[rank]
        assert y.shape == x.shape, (y.shape, x.shape)
        if not n:
            continue
        xr = x.reshape(n, H).contiguous()
        ridx, rwt = moe.gate(x)
        ridx, rwt = ridx.reshape(n, K).contiguous(), rwt.reshape(n, K).float().contiguous()
        want = torch.zeros_like(xr)
        native.check(lib.ktb200_moe_forward(full.handle, n, K, ridx.data_ptr(), rwt.data_ptr(), xr.data_ptr(), want.data_ptr(), None, s))
        for t0 in range(0, n, moe.BLOCK_MAX_TOKENS):     # the shared expert's handle takes BLOCK_MAX_TOKENS rows per call
            m = min(moe.BLOCK_MAX_TOKENS, n - t0)
            native.check(lib.ktb200_mlp_forward(moe._ktb_mlp, m, xr[t0:].data_ptr(), want[t0:].data_ptr(), 1, None, s))
        torch.cuda.synchronize()
        assert torch.equal(idx.reshape(n, K), ridx) and torch.equal(wt.reshape(n, K), rwt), f"rank {rank} step {st}: routing differs"
        ok, rel = bf16_close(y.reshape(n, H), want)
        assert ok, f"rank {rank} step {st} counts {counts}: rel err {rel:.2e}"
        worst = max(worst, rel)
    dist.barrier()
    print(f"rank {rank}/{world}: EP tokens OK over {len(steps)} steps, worst rel err {worst:.2e}", flush=True)
    torch.cuda.synchronize()
    os._exit(0)


if __name__ == "__main__":
    main()
