"""The Stable Diffusion VAE decoder's fused fp16 step on the H100 (sige_b200/workloads/sd_decoder.py, "mini": a 512-channel mid
block, so the D = 512 sparse-attention launch runs end to end): against the golden the reference's own SIGEDecoder produced,
graph replay against stream launches, and the next edit installed in place (set_masks, set_masks_async) against a fresh compile."""
import pytest
import torch

from conftest import golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _setup():
    from sige.utils import downsample_mask
    from sige_b200.workloads import sd_decoder as SD

    net = SD.build_sd_decoder("mini").to(DEV)
    z0, z1, mask = (t.to(DEV) for t in SD.sd_decoder_inputs("mini"))
    mask2 = torch.zeros_like(mask)
    mask2[12:20, 6:15] = True
    masks = [downsample_mask(m, min_res=(4, 4), dilation=0) for m in (mask, mask2)]
    with torch.no_grad():
        net.set_mode("full")
        net(z0)
        net.set_mode("sparse")
    return SD, net, z1, masks


def test_fused_step_matches_the_reference_golden_and_graph_replay_is_bitwise():
    from sige_b200.fused import FusedStep

    _, net, z1, masks = _setup()
    G = golden("sd_decoder_mini_golden.npz")
    with torch.no_grad():
        net.set_masks(masks[0])
        net.set_fused(True, dtype=torch.float16)
        out = net(z1).float()
        step = net.fused_step
        stream = FusedStep(net, z1, use_graph=False, dtype=torch.float16).output.clone()
        again = net(z1).clone()
    kinds = [k for k, _ in step.steps]
    ref = torch.from_numpy(G["sparse1"]).to(DEV)
    err = float((out - ref).abs().max() / ref.abs().max())
    print("sd decoder mini, fused fp16: %.3g of the golden's largest magnitude; %d tile convs, %d sparse-attention, eager %s"
          % (err, len(step.fused), kinds.count("sparse_attention"), step.eager_nodes))
    assert kinds.count("sparse_attention") == 1 and step.eager_nodes == []
    assert err <= 1e-2
    assert step.graph is not None and torch.equal(again.float(), out) and torch.equal(stream, again)


def test_next_edit_installs_in_place_like_a_fresh_compile():
    _, net, z1, masks = _setup()
    with torch.no_grad():
        net.set_fused(True, dtype=torch.float16)
        net.set_masks(masks[1])
        fresh = net(z1).clone()
        fresh_caps = sorted(sl.cap for sl in net.fused_step.low.slots.values())
        net.set_fused(True, dtype=torch.float16)
        net.set_masks(masks[0])
        net(z1)
        step = net.fused_step
        net.set_masks(masks[1])
        out_sync = net(z1).clone()
        assert net.fused_step is step, "the second edit fits: installed in place"
        net.set_masks(masks[0])
        net(z1)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            assert net.set_masks_async(masks[1]) is True
            out_async = net(z1).clone()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert net.fused_step is step and net.masks_async_ok()
        caps = sorted(sl.cap for sl in step.low.slots.values())
    assert torch.equal(out_async, out_sync), "device-installed lists == host-installed lists"
    d = float((out_sync.float() - fresh.float()).abs().max() / fresh.float().abs().max())
    print("in place vs fresh compile: %.3g (tile-list capacities %s, fresh %s)" % (d, caps, fresh_caps))
    if caps == fresh_caps:          # the same launch plans: the same bits
        assert torch.equal(out_sync, fresh)
    else:                           # other capacities may pick other split-K / cluster plans: fp16 reassociation only
        assert d <= 3e-3
