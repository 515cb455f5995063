"""Worker of tests/test_kquant_ep.py::test_ep_block_kquant_on_peer_memory (one process per GPU, torchrun): the one-launch
expert-parallel MoE block with Q2_K / Q3_K routed experts (argv[1]: "gate,up,down" ggml type ids) and a Q4_K / Q4_K / Q6_K
shared expert on REAL peer memory — every rank's token must equal the single-GPU layer over all experts (gate, routed
experts, then the shared expert as a second rounded term), over 12 back-to-back layers and CUDA-graph replays."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import gpu_util as G  # noqa: E402
from ktransformers_b200 import native  # noqa: E402
from ktransformers_b200.util.synth import synth_blocks  # noqa: E402
from oracle.bindings import BF16, Q4_K, Q6_K, bf16_to_f32, f32_to_bf16_bits  # noqa: E402

GT, UT, DT = (int(t) for t in sys.argv[1].split(","))


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    import torch.distributed._symmetric_memory as symm_mem
    lib = native.lib()
    E, k, H, I, ng, tg = 32, 4, 4096, 512, 4, 2
    El = E // world
    sy = lambda t, n, s: synth_blocks(t, n, device=dev, seed=s)
    gate_w, up_w, down_w = sy(GT, E * I * H, 401), sy(UT, E * I * H, 402), sy(DT, E * H * I, 403)
    sgs = (sy(Q4_K, I * H, 404), sy(Q4_K, I * H, 405), sy(Q6_K, H * I, 406))
    gb, db = gate_w.numel() // E, down_w.numel() // E
    rng = np.random.default_rng(7)
    Wr = rng.standard_normal((E, H)).astype(np.float32)
    bias = rng.standard_normal(E).astype(np.float32)
    gate = G.Gate(Wr, bias, k, ng, tg, hidden_type=BF16)
    full = G.Moe(E, k, H, I, gate_w.clone(), up_w.clone(), down_w.clone(), GT, UT, DT, BF16, max_tokens=8)
    full_mlp = G.Mlp(H, I, *(t.clone() for t in sgs), Q4_K, Q4_K, Q6_K, BF16)
    sl = slice(rank * El, (rank + 1) * El)
    shard = G.Moe(El, k, H, I, gate_w[sl.start * gb: sl.stop * gb].clone(), up_w[sl.start * gb: sl.stop * gb].clone(),
                  down_w[sl.start * db: sl.stop * db].clone(), GT, UT, DT, BF16, max_tokens=8, offset=sl.start)
    mlp = G.Mlp(H, I, *(t.clone() for t in sgs), Q4_K, Q4_K, Q6_K, BF16)
    msg_b, part_b, flag_b = world * lib.ktb200_ep_msg_bytes(H, BF16), world * H * 4, 4 * (2 * world + 2)
    o_part = (msg_b + 255) // 256 * 256
    o_flag = o_part + (part_b + 255) // 256 * 256
    sym = symm_mem.empty(o_flag + 256, dtype=torch.uint8, device=dev)
    sym.zero_()
    hdl = symm_mem.rendezvous(sym, dist.group.WORLD)
    base = [int(p) for p in hdl.buffer_ptrs]
    comm = native.EpComm.make(rank, world, H, BF16, base, [b + o_part for b in base], [b + o_flag for b in base])
    flags = sym[o_flag:o_flag + flag_b].view(torch.int32)
    torch.cuda.synchronize(); dist.barrier()
    y = torch.zeros((1, H), dtype=torch.bfloat16, device=dev)
    idx = torch.zeros((1, k), dtype=torch.int64, device=dev)
    w = torch.zeros((1, k), dtype=torch.float32, device=dev)
    x_d = torch.zeros((1, H), dtype=torch.bfloat16, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    worst = 0.0
    trng = np.random.default_rng(100 + rank)
    layers = 12
    xs = [f32_to_bf16_bits((trng.standard_normal((1, H)) / 10).astype(np.float32)) for _ in range(layers)]
    outs = []
    for l in range(layers):                       # back to back, no host synchronisation in between (buffer reuse across layers)
        x_d.copy_(G.dev(xs[l], torch.bfloat16))
        native.check(lib.ktb200_moe_ep_block_forward(C.byref(gate.cfg), shard.h, mlp.h, C.byref(comm), x_d.data_ptr(), y.data_ptr(),
                                                     idx.data_ptr(), w.data_ptr(), 7, s))
        outs.append((y.clone(), idx.clone(), w.clone()))
    torch.cuda.synchronize()
    assert int(flags[2 * world + 1]) == 0, "a peer wait timed out"
    for l in range(layers):
        want, widx, ww = G.moe_block_forward(gate, full, full_mlp, xs[l])
        yy, ii, wv = outs[l]
        assert np.array_equal(ii.cpu().numpy(), widx) and np.array_equal(wv.cpu().numpy(), ww), f"rank {rank} layer {l}: routing differs"
        a = bf16_to_f32(yy.cpu().view(torch.int16).numpy().view(np.uint16)); b = bf16_to_f32(want)
        err = np.abs(a - b)
        assert (err <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()).all(), f"rank {rank} layer {l}: max err {err.max()}"
        worst = max(worst, float(err.max() / np.abs(b).max()))
    # the same layers captured in ONE CUDA graph and replayed twice
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    dist.barrier()
    with torch.cuda.graph(g, stream=side):
        for l in range(4):
            native.check(lib.ktb200_moe_ep_block_forward(C.byref(gate.cfg), shard.h, mlp.h, C.byref(comm), x_d.data_ptr(), y.data_ptr(),
                                                         idx.data_ptr(), w.data_ptr(), 7, torch.cuda.current_stream().cuda_stream))
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    want, _, _ = G.moe_block_forward(gate, full, full_mlp, xs[-1])
    a = bf16_to_f32(y.cpu().view(torch.int16).numpy().view(np.uint16)); b = bf16_to_f32(want)
    assert (np.abs(a - b) <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()).all()
    assert int(flags[2 * world + 1]) == 0
    dist.barrier()
    print(f"rank {rank}/{world}: EP block OK over {layers} layers + graph replays, worst rel err {worst:.2e}", flush=True)
    torch.cuda.synchronize()
    os._exit(0)


if __name__ == "__main__":
    main()
