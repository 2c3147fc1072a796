"""GPU parity of the LiteFlowNet path (DeepModel.forward_flow, deep_models.py:144-182) through the
C ABI against the CPU oracle, on seeded synthetic weights / frames (oracle/synth.py)."""
import ctypes

import numpy as np
import pytest
import torch

from b200 import native
from oracle import nets, synth
from util import dptr, img_to_tensor

pytestmark = pytest.mark.gpu


def run_device(lib, H, W, ref, cur, prec, w):
    ctx = native.Context(lib)
    ctx.load_weights(native.NET_LITEFLOWNET, w)
    ctx.liteflow_build(H, W, 1, prec)
    d_ref, d_cur = torch.from_numpy(ref).cuda(), torch.from_numpy(cur).cuda()
    fwd = torch.zeros((2, H, W), dtype=torch.float32, device="cuda")
    bwd = torch.zeros_like(fwd)
    diff = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    ctx.liteflow_forward([d_ref.data_ptr(), d_cur.data_ptr()], dptr(fwd), dptr(bwd), dptr(diff))
    torch.cuda.synchronize()
    out = fwd.cpu().numpy(), bwd.cpu().numpy(), diff.cpu().numpy()
    ctx.close()
    return out


@pytest.mark.parametrize("H,W", [(70, 150), (128, 416)])
def test_liteflow_small_vs_oracle(dev_lib, H, W):
    ref, cur = synth.value_noise_image(H, W, 1), synth.value_noise_image(H, W, 2)
    w = synth.liteflownet_weights()
    with torch.no_grad():
        o = nets.liteflow_inference_flow(nets.to_torch(w), img_to_tensor(ref), img_to_tensor(cur))
    of, ob, od = o["forward"][0].numpy(), o["backward"][0].numpy(), o["flow_diff"][0, :, :, 0].numpy()
    # fp32 mode: summation-order differences only
    f, b, d = run_device(dev_lib, H, W, ref, cur, native.PREC_FP32, w)
    assert np.abs(f - of).max() < 2e-4 and np.abs(b - ob).max() < 2e-4 and np.abs(d - od).max() < 5e-4
    # bf16 tensor-core mode: flows of several px agree to a small fraction of a pixel (end-point error)
    f, b, d = run_device(dev_lib, H, W, ref, cur, native.PREC_BF16, w)
    epe = np.sqrt(((f - of) ** 2).sum(0))
    assert epe.mean() < 0.05 and epe.max() < 0.5, (epe.mean(), epe.max())
    assert np.abs(d - od).mean() < 0.08


def test_liteflow_full_size_properties(dev_lib):
    """BASELINE size 376x1241: no oracle run (minutes on CPU); size-independent properties instead:
    (1) swapping the two frames swaps forward and backward flow exactly (same kernels, same data);
    (2) identical frames through a symmetric path give fwd == bwd;
    (3) fp32 and bf16 modes agree to a fraction of a pixel."""
    H, W = 376, 1241
    ref, cur = synth.value_noise_image(H, W, 11), synth.value_noise_image(H, W, 12)
    w = synth.liteflownet_weights()
    f1, b1, d1 = run_device(dev_lib, H, W, ref, cur, native.PREC_BF16, w)
    f2, b2, d2 = run_device(dev_lib, H, W, cur, ref, native.PREC_BF16, w)
    assert np.array_equal(f1, b2) and np.array_equal(b1, f2)
    f3, b3, d3 = run_device(dev_lib, H, W, ref, ref, native.PREC_BF16, w)
    assert np.array_equal(f3, b3)
    assert np.isfinite(f1).all() and np.isfinite(d1).all()
    f4, b4, d4 = run_device(dev_lib, H, W, ref, cur, native.PREC_FP32, w)
    epe = np.sqrt(((f1 - f4) ** 2).sum(0))
    assert epe.mean() < 0.1, epe.mean()


def test_liteflow_two_pairs_batched(dev_lib):
    """Batched many-pairs mode (BASELINE configs[2] / SURVEY 8e): two independent pairs in one forward == each pair alone,
    bit for bit (wgmma path, bf16)."""
    H, W = 128, 416
    imgs = [synth.value_noise_image(H, W, s) for s in (1, 2, 3, 4)]
    w = synth.liteflownet_weights()

    def run(pairs, frames):
        ctx = native.Context(dev_lib)
        ctx.load_weights(native.NET_LITEFLOWNET, w)
        ctx.liteflow_build(H, W, pairs, native.PREC_BF16)
        d = [torch.from_numpy(f).cuda() for f in frames]
        fwd = torch.zeros((pairs, 2, H, W), dtype=torch.float32, device="cuda")
        bwd = torch.zeros_like(fwd)
        diff = torch.zeros((pairs, H, W), dtype=torch.float32, device="cuda")
        ctx.liteflow_forward([t.data_ptr() for t in d], dptr(fwd), dptr(bwd), dptr(diff))
        torch.cuda.synchronize()
        out = fwd.cpu().numpy(), bwd.cpu().numpy(), diff.cpu().numpy()
        ctx.close()
        return out

    f2, b2, d2 = run(2, imgs)
    for p in range(2):
        f1, b1, d1 = run(1, imgs[2 * p:2 * p + 2])
        assert np.array_equal(f2[p], f1[0]) and np.array_equal(b2[p], b1[0]) and np.array_equal(d2[p], d1[0]), p


def test_pair_batch_runner_matches_single_pairs(dev_lib):
    """b200.multi.PairBatchRunner (the per-rank unit of the sharded many-frames mode): its per-pair statistics equal those of
    the same pairs run one at a time."""
    from b200 import multi, runtime as rt_mod
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    H, W = 128, 416
    w = synth.liteflownet_weights()
    imgs = [rt.from_host(synth.value_noise_image(H, W, s)) for s in (1, 2, 3, 4, 5, 6)]
    all3 = multi.PairBatchRunner(rt, H, W, 3, w).forward(imgs)
    one = multi.PairBatchRunner(rt, H, W, 1, w)
    for p in range(3):
        assert np.array_equal(one.forward(imgs[2 * p:2 * p + 2])[0], all3[p]), p
    assert all3.shape == (3, 2) and (all3[:, 0] > 0).all()


def test_layer_chains_bit_equal_to_per_layer_launches(dev_lib):
    """csrc/conv_chain.cu (opt-in, dfvo_set_conv_chain / DFVO_CONV_CHAIN=1): the chained launch walks the same K order per output
    element as the per-layer kernels, so both flows and the consistency map must be bit-identical, at the BASELINE size (all five
    levels, chains of 3..9 layers) and at a small ragged size."""
    w = synth.liteflownet_weights()
    prev = dev_lib.dfvo_set_conv_chain(0)
    try:
        for H, W, seed in [(376, 1241, 21), (70, 150, 23)]:
            ref, cur = synth.value_noise_image(H, W, seed), synth.value_noise_image(H, W, seed + 1)
            dev_lib.dfvo_set_conv_chain(0)
            n0 = dev_lib.dfvo_launch_count()
            a = run_device(dev_lib, H, W, ref, cur, native.PREC_BF16, w)
            n1 = dev_lib.dfvo_launch_count()
            dev_lib.dfvo_set_conv_chain(1)
            b = run_device(dev_lib, H, W, ref, cur, native.PREC_BF16, w)
            n2 = dev_lib.dfvo_launch_count()
            assert (n2 - n1) < (n1 - n0) - 30, (n1 - n0, n2 - n1)          # the chains really replaced launches
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
    finally:
        dev_lib.dfvo_set_conv_chain(prev)
