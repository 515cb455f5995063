"""Minimal DeepSeek-V3 MoE block definitions — the injection targets of the H100 rule files.

Only the classes the hot path's YAML rules match against are defined here (the reference carries the
whole HF model, archive/ktransformers/models/modeling_deepseek_v3.py; everything outside the MoE block
is out of scope, SURVEY §2.2).  Semantics restate the reference:
    DeepseekV3MLP   :385-397     down(silu(gate x) * up x)
    MoEGate         :400-481     sigmoid scoring + noaux_tc grouped top-k
    DeepseekV3MoE   :483-616     gate -> routed experts (+ shared experts)
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn
from transformers.configuration_utils import PretrainedConfig


class DeepseekV3Config(PretrainedConfig):
    model_type = "deepseek_v3"

    def __init__(self, hidden_size=7168, intermediate_size=18432, moe_intermediate_size=2048, n_routed_experts=256,
                 n_shared_experts=1, num_experts_per_tok=8, n_group=8, topk_group=4, routed_scaling_factor=2.5,
                 norm_topk_prob=True, scoring_func="sigmoid", topk_method="noaux_tc", hidden_act="silu",
                 num_hidden_layers=61, first_k_dense_replace=3, moe_layer_freq=1, num_attention_heads=128,
                 q_lora_rank=1536, kv_lora_rank=512, qk_rope_head_dim=64, qk_nope_head_dim=128, v_head_dim=128,
                 vocab_size=129280, rms_norm_eps=1e-6, ep_size=1, **kwargs):
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.moe_intermediate_size = moe_intermediate_size
        self.n_routed_experts = n_routed_experts
        self.n_shared_experts = n_shared_experts
        self.num_experts_per_tok = num_experts_per_tok
        self.n_group = n_group
        self.topk_group = topk_group
        self.routed_scaling_factor = routed_scaling_factor
        self.norm_topk_prob = norm_topk_prob
        self.scoring_func = scoring_func
        self.topk_method = topk_method
        self.hidden_act = hidden_act
        self.num_hidden_layers = num_hidden_layers
        self.first_k_dense_replace = first_k_dense_replace
        self.moe_layer_freq = moe_layer_freq
        self.num_attention_heads = num_attention_heads
        self.q_lora_rank = q_lora_rank
        self.kv_lora_rank = kv_lora_rank
        self.qk_rope_head_dim = qk_rope_head_dim
        self.qk_nope_head_dim = qk_nope_head_dim
        self.v_head_dim = v_head_dim
        self.vocab_size = vocab_size
        self.rms_norm_eps = rms_norm_eps
        self.ep_size = ep_size
        super().__init__(**kwargs)


class DeepseekV3MLP(nn.Module):
    def __init__(self, config, hidden_size=None, intermediate_size=None):
        super().__init__()
        self.config = config
        self.hidden_size = hidden_size or config.hidden_size
        self.intermediate_size = intermediate_size or config.intermediate_size
        self.gate_proj = nn.Linear(self.hidden_size, self.intermediate_size, bias=False)
        self.up_proj = nn.Linear(self.hidden_size, self.intermediate_size, bias=False)
        self.down_proj = nn.Linear(self.intermediate_size, self.hidden_size, bias=False)
        self.act_fn = F.silu

    def forward(self, x):
        return self.down_proj(self.act_fn(self.gate_proj(x)) * self.up_proj(x))


class MoEGate(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.top_k = config.num_experts_per_tok
        self.n_routed_experts = config.n_routed_experts
        self.routed_scaling_factor = config.routed_scaling_factor
        self.scoring_func = config.scoring_func
        self.topk_method = config.topk_method
        self.n_group = config.n_group
        self.topk_group = config.topk_group
        self.norm_topk_prob = config.norm_topk_prob
        self.gating_dim = config.hidden_size
        self.weight = nn.Parameter(torch.empty((self.n_routed_experts, self.gating_dim)))
        if self.topk_method == "noaux_tc":
            self.e_score_correction_bias = nn.Parameter(torch.empty((self.n_routed_experts)))
        if self.weight.device.type != "meta":
            nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
            if self.topk_method == "noaux_tc":
                nn.init.zeros_(self.e_score_correction_bias)

    def forward(self, hidden_states):
        bsz, seq_len, h = hidden_states.shape
        x = hidden_states.view(-1, h)
        logits = F.linear(x.type(torch.float32), self.weight.type(torch.float32), None)
        if self.scoring_func != "sigmoid":
            raise NotImplementedError(f"insupportable scoring function for MoE gating: {self.scoring_func}")
        scores = logits.sigmoid()
        if self.topk_method != "noaux_tc":
            raise NotImplementedError(f"insupportable TopK function for MoE gating: {self.topk_method}")
        n = bsz * seq_len
        choice = scores.view(n, -1) + self.e_score_correction_bias.unsqueeze(0)
        group_scores = choice.view(n, self.n_group, -1).topk(2, dim=-1)[0].sum(dim=-1)
        group_idx = torch.topk(group_scores, k=self.topk_group, dim=-1, sorted=False)[1]
        group_mask = torch.zeros_like(group_scores)
        group_mask.scatter_(1, group_idx, 1)
        score_mask = group_mask.unsqueeze(-1).expand(n, self.n_group, self.n_routed_experts // self.n_group).reshape(n, -1)
        tmp = choice.masked_fill(~score_mask.bool(), float("-inf"))
        _, topk_idx = torch.topk(tmp, k=self.top_k, dim=-1, sorted=False)
        topk_weight = scores.gather(1, topk_idx)
        if self.top_k > 1 and self.norm_topk_prob:
            topk_weight = topk_weight / (topk_weight.sum(dim=-1, keepdim=True) + 1e-20)
        topk_weight = topk_weight * self.routed_scaling_factor
        return topk_idx, topk_weight


class DeepseekV3MoE(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.num_experts_per_tok = config.num_experts_per_tok
        self.ep_size, self.experts_per_rank, self.ep_rank = 1, config.n_routed_experts, 0
        self.experts = nn.ModuleList([DeepseekV3MLP(config, intermediate_size=config.moe_intermediate_size)
                                      for _ in range(config.n_routed_experts)])
        self.gate = MoEGate(config)
        if config.n_shared_experts is not None:
            self.shared_experts = DeepseekV3MLP(config, intermediate_size=config.moe_intermediate_size * config.n_shared_experts)

    def forward(self, hidden_states):
        identity = hidden_states
        orig_shape = hidden_states.shape
        topk_idx, topk_weight = self.gate(hidden_states)
        x = hidden_states.view(-1, hidden_states.shape[-1])
        y = torch.zeros_like(x)
        for t in range(x.shape[0]):
            for j in range(topk_idx.shape[1]):
                y[t] += self.experts[int(topk_idx[t, j])](x[t]) * topk_weight[t, j].to(x.dtype)
        y = y.view(*orig_shape)
        if self.config.n_shared_experts is not None:
            y = y + self.shared_experts(identity)
        return y


class DeepseekV3RMSNorm(nn.Module):
    """modeling_deepseek_v3.py:65-80: fp32 variance, weight applied in the input dtype."""

    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, hidden_states):
        input_dtype = hidden_states.dtype
        h = hidden_states.to(torch.float32)
        h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + self.variance_epsilon)
        return self.weight * h.to(input_dtype)


def yarn_get_mscale(scale=1.0, mscale=1.0):
    return 1.0 if scale <= 1 else 0.1 * mscale * math.log(scale) + 1.0


class DeepseekV3RotaryEmbedding(nn.Module):
    """Plain RoPE tables (modeling_deepseek_v3.py:100-140); `forward(x, position_ids)` returns (cos, sin) [bsz, q_len, dim]
    the way the injected YarnRotaryEmbeddingV3 does (operators/RoPE.py:222-326)."""

    def __init__(self, dim, max_position_embeddings=163840, base=10000.0):
        super().__init__()
        self.dim, self.base = dim, base
        inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim))
        self.register_buffer("inv_freq", inv_freq, persistent=False)

    @torch.no_grad()
    def forward(self, x, position_ids):
        freqs = position_ids[:, :, None].float() * self.inv_freq.to(position_ids.device)[None, None, :]
        emb = torch.cat((freqs, freqs), dim=-1)
        return emb.cos().to(x.dtype), emb.sin().to(x.dtype)


def rotate_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def apply_rotary_pos_emb(q, k, cos, sin, unsqueeze_dim=1):
    """modeling_deepseek_v3.py:339-373, including the de-interleaving permutation of the rope dims."""
    cos, sin = cos.unsqueeze(unsqueeze_dim), sin.unsqueeze(unsqueeze_dim)
    b, s, h, d = q.shape
    q = q.view(b, s, h, d // 2, 2).transpose(4, 3).reshape(b, s, h, d)
    b, s, h, d = k.shape
    k = k.view(b, s, h, d // 2, 2).transpose(4, 3).reshape(b, s, h, d)
    return (q * cos) + (rotate_half(q) * sin), (k * cos) + (rotate_half(k) * sin)


class DeepseekV3Attention(nn.Module):
    """Multi-head latent attention, modeling_deepseek_v3.py:619-800: the injection target of KDeepseekV2Attention.  `forward`
    here is the plain (non-absorbed, full-precision) formulation over an explicit list of past latents — the restatement
    the operator tests compare the absorbed paged decode against."""

    def __init__(self, config, layer_idx: int = 0):
        super().__init__()
        self.config, self.layer_idx = config, layer_idx
        self.hidden_size, self.num_heads = config.hidden_size, config.num_attention_heads
        self.q_lora_rank, self.kv_lora_rank = config.q_lora_rank, config.kv_lora_rank
        self.qk_rope_head_dim, self.qk_nope_head_dim, self.v_head_dim = config.qk_rope_head_dim, config.qk_nope_head_dim, config.v_head_dim
        self.q_head_dim = self.qk_nope_head_dim + self.qk_rope_head_dim
        if self.q_lora_rank is None:
            self.q_proj = nn.Linear(self.hidden_size, self.num_heads * self.q_head_dim, bias=False)
        else:
            self.q_a_proj = nn.Linear(self.hidden_size, self.q_lora_rank, bias=False)
            self.q_a_layernorm = DeepseekV3RMSNorm(self.q_lora_rank, config.rms_norm_eps)
            self.q_b_proj = nn.Linear(self.q_lora_rank, self.num_heads * self.q_head_dim, bias=False)
        self.kv_a_proj_with_mqa = nn.Linear(self.hidden_size, self.kv_lora_rank + self.qk_rope_head_dim, bias=False)
        self.kv_a_layernorm = DeepseekV3RMSNorm(self.kv_lora_rank, config.rms_norm_eps)
        self.kv_b_proj = nn.Linear(self.kv_lora_rank, self.num_heads * (self.qk_nope_head_dim + self.v_head_dim), bias=False)
        self.o_proj = nn.Linear(self.num_heads * self.v_head_dim, self.hidden_size, bias=False)
        self.rotary_emb = DeepseekV3RotaryEmbedding(self.qk_rope_head_dim, base=getattr(config, "rope_theta", 10000.0))
        self.softmax_scale = self.q_head_dim ** (-0.5)
        rs = getattr(config, "rope_scaling", None)
        if rs is not None and rs.get("mscale_all_dim", 0):
            m = yarn_get_mscale(rs["factor"], rs["mscale_all_dim"])
            self.softmax_scale = self.softmax_scale * m * m

    def project(self, hidden_states, position_ids):
        """(q_nope [b,s,h,128], q_pe [b,s,h,64] roped, ckv [b,s,1,512] normed, k_pe [b,s,1,64] roped)"""
        bsz, q_len, _ = hidden_states.size()
        q = self.q_proj(hidden_states) if self.q_lora_rank is None else self.q_b_proj(self.q_a_layernorm(self.q_a_proj(hidden_states)))
        q = q.view(bsz, q_len, self.num_heads, self.q_head_dim)
        q_nope, q_pe = torch.split(q, [self.qk_nope_head_dim, self.qk_rope_head_dim], dim=-1)
        ckv = self.kv_a_proj_with_mqa(hidden_states)
        ckv, k_pe = torch.split(ckv, [self.kv_lora_rank, self.qk_rope_head_dim], dim=-1)
        ckv = self.kv_a_layernorm(ckv).view(bsz, q_len, 1, self.kv_lora_rank)
        k_pe = k_pe.view(bsz, q_len, 1, self.qk_rope_head_dim)
        cos, sin = self.rotary_emb(q_pe, position_ids)
        q_pe, k_pe = apply_rotary_pos_emb(q_pe, k_pe, cos, sin, unsqueeze_dim=2)
        return q_nope, q_pe, ckv, k_pe

    def forward(self, hidden_states, position_ids, past_latents=None):
        """past_latents: optional (ckv [b, L, 512], k_pe [b, L, 64]) of the earlier tokens; causal within the new tokens."""
        bsz, q_len, _ = hidden_states.size()
        q_nope, q_pe, ckv, k_pe = self.project(hidden_states, position_ids)
        ckv, k_pe = ckv.squeeze(2), k_pe.squeeze(2)
        if past_latents is not None:
            ckv, k_pe = torch.cat([past_latents[0], ckv], 1), torch.cat([past_latents[1], k_pe], 1)
        L = ckv.shape[1]
        kv = self.kv_b_proj(ckv).view(bsz, L, self.num_heads, self.qk_nope_head_dim + self.v_head_dim)
        k_nope, v = torch.split(kv, [self.qk_nope_head_dim, self.v_head_dim], dim=-1)
        s = torch.einsum("bqhd,bkhd->bhqk", q_nope.float(), k_nope.float()) + torch.einsum("bqhd,bkd->bhqk", q_pe.float(), k_pe.float())
        s = s * self.softmax_scale
        mask = torch.arange(L, device=s.device)[None, :] > (L - q_len + torch.arange(q_len, device=s.device))[:, None]
        s = s.masked_fill(mask[None, None], float("-inf"))
        o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v.float()).to(hidden_states.dtype)
        return self.o_proj(o.reshape(bsz, q_len, self.num_heads * self.v_head_dim)), (ckv, k_pe)


class DeepseekV3DecoderLayerMoEOnly(nn.Module):
    """A decoder layer reduced to its MoE block (what the hot path covers)."""

    def __init__(self, config, layer_idx: int):
        super().__init__()
        dense = layer_idx < config.first_k_dense_replace
        self.mlp = DeepseekV3MLP(config) if dense else DeepseekV3MoE(config)

    def forward(self, hidden_states):
        return hidden_states + self.mlp(hidden_states)


class DeepseekV3MoEStack(nn.Module):
    """`model.layers.N.mlp` naming so that GGUF keys (`blk.N.ffn_*`) and rule regexes line up with the
    reference's full model."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.layers = nn.ModuleList([DeepseekV3DecoderLayerMoEOnly(config, i) for i in range(config.num_hidden_layers)])

    def forward(self, hidden_states):
        for layer in self.layers:
            hidden_states = layer(hidden_states)
        return hidden_states


class DeepseekV3MoEOnlyForCausalLM(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.model = DeepseekV3MoEStack(config)
        self.lm_head = nn.Identity()

    def forward(self, hidden_states):
        return self.model(hidden_states)
