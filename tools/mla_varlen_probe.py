"""The attention core of a ragged step with prompt chunks: every row absorbed (today's forward_ragged) against the split
of forward_ragged without absorb_for_prefill (gather + kv_b_proj + ktb200_mla_prefill_varlen for the prompt sequences, the
absorbed branch for the decode rows), on one GPU.

(a) 7 decode rows at 4096..32768 cached tokens and one 512-token prompt chunk at P = 0 (DESIGN §4.16's batch);
(b) four new 1024-token prompts;
(c) two decode rows at 32768, a 2048-token chunk at P = 4096 and a new 150-token prompt.
Absorbed = absorb_q over all rows, the ragged MLAWrapper plan and run, absorb_o; split = KDeepseekV2Attention._ragged_split.
Both start from the same q_b output, roped q_pe and latent cache, and both include their host work (plans, index copies).
Also the varlen kernel alone against one ktb200_mla_prefill call per prompt sequence, on the same decompressed operands.
V3 shapes (128 heads, 512 + 64 latent, pages of 64).  CUDA-event windows of >= 50 ms, the median of 3 alternating rounds.
The card's name and power limit are read in the same run.

    python tools/mla_varlen_probe.py [--out results.json]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ktransformers_b200 import native  # noqa: E402
from ktransformers_b200.models.custom_cache import StaticCache  # noqa: E402
from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Attention, DeepseekV3Config  # noqa: E402
from ktransformers_b200.operators import attention as attn_mod  # noqa: E402
from ktransformers_b200.operators.attention import KDeepseekV2Attention  # noqa: E402
from mla_ragged_probe import card, median_alternating  # noqa: E402

H = 128


class Step:
    """one ragged step's operands after the projections and the cache write: sequences b at cache rows b"""

    def __init__(self, op, cfg, q_lens, kv_len, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.op = op
        self.q_lens, self.kv_len = np.array(q_lens, np.int32), np.array(kv_len, np.int32)
        B, T = len(q_lens), int(sum(q_lens))
        self.cache = StaticCache(cfg, max_batch_size=B, max_cache_len=int(self.kv_len.max()), device="cuda")
        lat = self.cache.key_cache[0]
        lat.copy_(torch.randn(lat.shape, generator=g, device="cuda").to(torch.bfloat16))
        self.q = (torch.randn((1, T, H, 192), generator=g, device="cuda") * 0.5).to(torch.bfloat16)
        self.q_pe = (torch.randn((T, H, 64), generator=g, device="cuda") * 0.5).to(torch.bfloat16)
        self.qo = torch.from_numpy(np.r_[0, np.cumsum(self.q_lens)].astype(np.int32))
        self.kl = torch.from_numpy(self.kv_len)
        self.rows = torch.arange(B, dtype=torch.int32)
        self.T, self.B = T, B

    def split(self):
        return self.op._ragged_split(self.q, self.q_pe, self.cache.key_cache[0], self.qo, self.kl, self.rows, self.cache, 4096, 16384)

    def absorbed(self):
        """forward_ragged's absorbed branch, from absorb_q to absorb_o"""
        op, T, dev = self.op, self.T, self.q.device
        lib, stream = native.lib(), torch.cuda.current_stream().cuda_stream
        q_absorb, out_absorb = op.get_absorbed()
        q_abs = torch.empty((T, H, 512), dtype=torch.bfloat16, device=dev)
        native.check(lib.ktb200_mla_absorb_q(self.q.data_ptr(), 192, H * 192, q_absorb.data_ptr(), H, 128, 512, q_abs.data_ptr(), T, stream))
        w = attn_mod._ragged_wrapper(self.cache, dev, self.B, 4096, 16384)
        kv_indptr = torch.arange(0, self.B + 1, dtype=torch.int32, device=dev) * self.cache.max_pages
        kv_indices = self.cache.page_table_list[0].index_select(0, self.rows.to(dev).long()).reshape(-1)
        w.plan(self.qo, kv_indptr, kv_indices, self.kl, None, H, 512, 64, 64, op.softmax_scale, torch.bfloat16, torch.bfloat16)
        kv = self.cache.key_cache[0]
        attn = w.run(q_abs, self.q_pe, kv[..., :512].view(-1, 64, 512), kv[..., 512:].view(-1, 64, 64))
        o = torch.empty((T, H, 128), dtype=torch.bfloat16, device=dev)
        native.check(lib.ktb200_mla_absorb_o(attn.data_ptr(), out_absorb.data_ptr(), H, 128, 512, o.data_ptr(), T, stream))
        return o

    def kernels(self):
        """(one varlen call, one ktb200_mla_prefill per prompt sequence) on the decompressed operands of the prompt sequences"""
        lib, stream = native.lib(), torch.cuda.current_stream().cuda_stream
        pre = [b for b in range(self.B) if self.q_lens[b] > 1]
        n = int(self.kv_len[pre].sum())
        lat = torch.cat([self.cache.key_cache[0].view(self.B, -1, 576)[b, :int(self.kv_len[b])] for b in pre])
        kv = self.op.kv_b_proj(lat[:, :512]).view(n, H, 256)
        qn, kn, v, kp = self.q[0, ..., :128], kv[..., :128], kv[..., 128:], lat[:, 512:]
        starts = np.r_[0, np.cumsum(self.kv_len[pre])[:-1]]
        seq = np.ascontiguousarray(np.stack([self.qo.numpy()[pre], self.q_lens[pre], starts, self.kv_len[pre]], 1).astype(np.int32))
        out_v = torch.empty((self.T, H, 128), dtype=torch.bfloat16, device="cuda")
        pv = native.MlaPrefillVarlenParams(len(pre), self.T, n, H, 128, 64, 128, self.op.softmax_scale, seq.ctypes.data, qn.data_ptr(), qn.stride(0),
                                           qn.stride(1), self.q_pe.data_ptr(), self.q_pe.stride(0), self.q_pe.stride(1), kn.data_ptr(), kn.stride(0),
                                           kn.stride(1), v.data_ptr(), v.stride(0), v.stride(1), kp.data_ptr(), kp.stride(0), out_v.data_ptr())
        out_d = torch.empty_like(out_v)
        dense = []
        for (qr, ql, kr, kl) in seq.tolist():
            a, b = qn[qr:qr + ql], self.q_pe[qr:qr + ql]
            big = 1 << 30
            dense.append(native.MlaPrefillParams(1, ql, kl, H, 128, 64, 128, self.op.softmax_scale, a.data_ptr(), a.stride(0), a.stride(1), big,
                                                 b.data_ptr(), b.stride(0), b.stride(1), big, kn[kr].data_ptr(), kn.stride(0), kn.stride(1), big,
                                                 v[kr].data_ptr(), v.stride(0), v.stride(1), big, kp[kr].data_ptr(), kp.stride(0), big,
                                                 out_d[qr].data_ptr()))
        keep = (seq, kv, lat, out_v, out_d, pv, dense)
        varlen = lambda: native.check(lib.ktb200_mla_prefill_varlen(C.byref(keep[5]), stream))
        separate = lambda: [native.check(lib.ktb200_mla_prefill(C.byref(p), stream)) for p in keep[6]]
        rows = torch.cat([torch.arange(int(r), int(r) + int(q)) for r, q in zip(seq[:, 0], seq[:, 1])]).cuda()
        return varlen, separate, out_v, out_d, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times the GPU; there is nothing to measure without one"
    torch.manual_seed(0)
    cfg = DeepseekV3Config(hidden_size=1024, num_attention_heads=H, q_lora_rank=256, num_hidden_layers=1)
    plain = DeepseekV3Attention(cfg, layer_idx=0).to(device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        plain.kv_b_proj.weight.normal_(0, 512 ** -0.5)
    op = KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda")
    res = {"card": card(), "heads": H, "page_size": 64}
    batches = {"a_7_decode_plus_512_chunk": ([1, 1, 512, 1, 1, 1, 1, 1], [4096, 8192, 512, 12288, 16384, 20480, 24576, 32768]),
               "b_four_1024_prompts": ([1024] * 4, [1024] * 4),
               "c_2_decode_2048_chunk_150_prompt": ([1, 1, 2048, 150], [32768, 32768, 4096 + 2048, 150])}
    with torch.no_grad():
        for i, (name, (q, kv)) in enumerate(batches.items()):
            attn_mod._RAGGED_WRAPPERS.clear()
            st = Step(op, cfg, q, kv, seed=i + 1)
            t = median_alternating({"absorbed": st.absorbed, "split": st.split})
            diff = (st.absorbed().float() - st.split().float()).abs()
            ref = st.absorbed().float().abs().max().item()
            varlen, separate, out_v, out_d, rows = st.kernels()
            k = median_alternating({"varlen": varlen, "separate": separate})
            torch.cuda.synchronize()
            res[name] = {"absorbed_ms": t["absorbed"], "split_ms": t["split"], "speedup": t["absorbed"] / t["split"],
                         "max_abs_diff": diff.max().item(), "max_abs_out": ref,
                         "varlen_kernel_ms": k["varlen"], "separate_prefill_calls_ms": k["separate"],
                         "varlen_equals_separate": bool(torch.equal(out_v[rows].view(torch.int16), out_d[rows].view(torch.int16)))}
            print(name, json.dumps(res[name]), flush=True)
            del st
            torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
