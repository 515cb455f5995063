"""The persistent MoE-block kernel hands the intermediate activations from gate/up to down through per-Q8_K-block
readiness words instead of a grid barrier.  Every launch must leave those words, the grid-barrier words and the
timeout status word at zero, whatever the launch mode, and give the bits of the separate launches."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sync_words(moe):
    import ctypes as C

    from ktransformers_b200 import native
    lib = native.lib()
    n = lib.ktb200_debug_block_sync_words(moe.h, None, 0)
    assert n > 8
    buf = (C.c_uint * n)()
    assert lib.ktb200_debug_block_sync_words(moe.h, buf, n) == n
    return np.frombuffer(buf, dtype=np.uint32)


def _mixed_launches():
    """Two handles of different shapes (with and without a shared expert, Q6_K and Q4_K down), interleaved back to back
    at several token counts, then in a captured graph; returns (what went wrong, or None)."""
    import torch

    import gpu_util as G
    from ktransformers_b200 import native
    from ktransformers_b200.util.synth import synth_blocks
    from oracle.bindings import BF16, Q4_K, Q6_K, f32_to_bf16_bits

    torch.cuda.set_device(0)
    rng = np.random.default_rng(7)
    Eg, k = 16, 4
    hs = []
    for i, (H, I, dt, shared) in enumerate([(4096, 512, Q6_K, True), (4096, 2048, Q4_K, False)]):
        s = lambda t, n, j: synth_blocks(t, n, device="cuda", seed=100 * i + j)  # noqa: E731
        m = G.Moe(Eg, k, H, I, s(Q4_K, Eg * I * H, 1), s(Q4_K, Eg * I * H, 2), s(dt, Eg * H * I, 3), Q4_K, Q4_K, dt, BF16, max_tokens=8)
        mlp = G.Mlp(H, I, s(Q4_K, I * H, 4), s(Q4_K, I * H, 5), s(dt, H * I, 6), Q4_K, Q4_K, dt, BF16) if shared else None
        gate = G.Gate(rng.standard_normal((Eg, H)).astype(np.float32), rng.standard_normal(Eg).astype(np.float32), k, 4, 2, hidden_type=BF16)
        hs.append((gate, m, mlp, H))
    for qlen in (1, 8, 3):
        for gate, m, mlp, H in hs:
            x = f32_to_bf16_bits((rng.standard_normal((qlen, H)) / 10).astype(np.float32))
            n0 = native.launch_count()
            out, idx, w = G.moe_block_forward(gate, m, mlp, x, repeats=3)
            if native.launch_count() - n0 != 3:
                return "the persistent kernel did not take the call"
            want = G.moe_forward_shared(m, mlp, idx, w, x)
            if not np.array_equal(out, want):
                return f"qlen={qlen} H={H}: not bit-identical to the separate launches"
            replay = G.moe_block_forward(gate, m, mlp, x, repeats=3, graph=True)
            if not all(np.array_equal(a, b) for a, b in zip((out, idx, w), replay)):
                return f"qlen={qlen} H={H}: graph replay differs"
    for gate, m, mlp, H in hs:
        words = _sync_words(m)
        if words[4] != 0:
            return "a readiness wait timed out"
        if words.any():
            return f"synchronisation words left non-zero at {np.nonzero(words)[0][:8].tolist()}"
        m.close()
        if mlp is not None:
            mlp.close()
    return None


@pytest.mark.gpu
def test_sync_words_are_zero_after_mixed_launches_and_graph_replays():
    err = _mixed_launches()
    assert err is None, err


# the launch-mode variables are read once per process: each mode runs in its own interpreter
@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"KTB200_BLK_COOP": "0"}, {"KTB200_BLK_WARPS": "15"}, {"KTB200_BLK_COOP": "0", "KTB200_BLK_WARPS": "15"}])
def test_sync_words_are_zero_in_other_launch_modes(env):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env={**os.environ, **env})
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]


if __name__ == "__main__":
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    err = _mixed_launches()
    print(err if err else "OK")
    sys.exit(1 if err else 0)
