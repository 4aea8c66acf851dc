"""DROID-style plugin surface on the GPU (nerf_slam_b200/droid.py): operator adapter parity, FactorGraph.update
against the validated RaftVisualFrontend building blocks, and the MotionFilter + DroidFrontend loop end to end.

"""
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = os.path.join(ROOT, "oracle", "_ref", "droid.pth")
DEV = "cuda:0"


def _net():
    from nerf_slam_b200.droid import DroidNet
    return DroidNet(WEIGHTS if os.path.exists(WEIGHTS) else None, DEV)


def test_update_net_reference_convention_matches_library():
    """UpdateNetTC (wgmma) vs the library-convolution UpdateModule on the reference's tensor layouts;
    tolerances of tests/test_gpu_conv.py (fp16 operands, different summation order)"""
    net = _net()
    g = torch.Generator(device=DEV).manual_seed(5)
    E, h, w = 5, 30, 40
    r = lambda *s: torch.randn(*s, generator=g, device=DEV)
    hid = torch.tanh(r(1, E, 128, h, w)).half(); inp = torch.relu(r(1, E, 128, h, w)).half()
    corr = (0.5 * r(1, E, 196, h, w)).half(); motion = (2.0 * r(1, E, 4, h, w)).clamp(-64, 64)
    ii = torch.tensor([0, 0, 1, 3, 3], device=DEV)
    got = net.update_net(hid, inp, corr, motion, ii, ii)
    ref = net.update_net.params(hid, inp, corr, motion.half(), ii, ii)
    assert got[0].shape == ref[0].shape == (1, E, 128, h, w)
    assert (got[0].float() - ref[0].float()).abs().max() < 3e-2        # tolerances of tests/test_gpu_conv.py (fp16 state)
    assert (got[1] - ref[1].float()).abs().max() < 6e-2
    assert (got[2] - ref[2].float()).abs().max() < 2e-3
    assert got[3].shape == ref[3].shape == (1, 3, h, w)
    assert (got[3] - ref[3].float()).abs().max() < 2e-3
    assert got[4].shape == ref[4].shape == (1, 3, 576, h, w)
    assert (got[4].float() - ref[4].float()).abs().max() < 5e-2
    out3 = net.update_net(hid[:, :1], inp[:, :1], corr[:, :1])                 # MotionFilter's call (no flow, no ii)
    assert len(out3) == 3 and out3[1].shape == (1, 1, h, w, 2)


def _filled_video(n=8, H=240, W=320, step=0.03):
    """video filled by the MotionFilter from the procedural stream, depths/poses perturbed from ground truth"""
    from nerf_slam_b200.droid import DepthVideo, MotionFilter
    from nerf_slam_b200.synthetic import SyntheticRoom
    net = _net()
    room = SyntheticRoom(W, H, 200, seed=0, step=step)
    video = DepthVideo((H, W), buffer=32, device=DEV)
    filt = MotionFilter(net, video, min_flow_thresh=2.4, device=DEV)
    k = 0
    while video.counter.value < n and k < 200:
        p = room.packet(k)
        img = torch.as_tensor(np.asarray(p["images"]))[..., [2, 1, 0]].permute(0, 3, 1, 2).contiguous()   # RGB(A) -> BGR, [1,3,H,W]
        filt.track(k, float(p["t_cams"][0]), img, None, torch.as_tensor(p["calibs"][0].camera_model.numpy()))
        k += 1
    assert video.counter.value == n, "motion filter kept too few frames"
    return net, video, room


def test_factor_graph_update_moves_towards_consistency():
    """16 updates on a neighbourhood graph (DroidFrontend.__initialize's first half): finite state, valid unit
    quaternions, positive depths, graph invariants, and a flow residual that shrinks"""
    from nerf_slam_b200.droid import FactorGraph
    net, video, room = _filled_video()
    graph = FactorGraph(video, net.update_net, device=DEV, max_factors=48, upsample=True)
    graph.add_neighborhood_factors(0, video.counter.value, r=3)
    E = len(graph.ii)
    assert graph.gru_hidden_states.shape == (1, E, 128, 30, 40) and graph.gru_contexts_input.shape == (1, E, 128, 30, 40)
    res = []
    for _ in range(8):
        graph.update(1, use_inactive=True)
        coords1, _ = video.reproject(graph.ii, graph.jj)
        res.append(float((graph.gru_estimated_flow - coords1).abs().mean()))
    torch.cuda.synchronize()
    n = video.counter.value
    assert torch.isfinite(video.poses[:n]).all() and torch.isfinite(video.disps[:n]).all()
    assert (video.disps[:n] >= 1e-3).all()
    assert torch.allclose(video.poses[:n, 3:].norm(dim=-1), torch.ones(n, device=DEV), atol=1e-4)
    assert video.poses[0].tolist() == [0, 0, 0, 0, 0, 0, 1]                      # t0 = 1: the first pose is the gauge
    assert graph.age.tolist() == [8] * E
    if os.path.exists(WEIGHTS):                                                  # trained operator: BA and flow converge
        assert res[-1] < res[0], f"flow residual did not shrink: {res}"
    assert torch.isfinite(video.disps_up[:n]).all() and video.disps_up[1].abs().sum() > 0


def test_factor_graph_generic_callable_matches_fused_path():
    """FactorGraph with a plain reference-convention callable (the library UpdateModule) and with the fused
    operator must produce the same flow/confidence after one update from the same state"""
    from nerf_slam_b200.droid import FactorGraph
    net, video, room = _filled_video(6)
    outs = []
    for update_net in (net.update_net, net.update_net.params):
        graph = FactorGraph(video, update_net, device=DEV, max_factors=48)
        graph.add_neighborhood_factors(0, video.counter.value, r=2)
        poses, disps = video.poses.clone(), video.disps.clone()
        graph.update(1, use_inactive=False)
        outs.append((graph.gru_estimated_flow.clone(), graph.gru_estimated_flow_weight.clone(), graph.gru_hidden_states.float().clone()))
        video.poses.copy_(poses); video.disps.copy_(disps)
    assert (outs[0][0] - outs[1][0]).abs().max() < 6e-2
    assert (outs[0][1] - outs[1][1]).abs().max() < 2e-2
    assert (outs[0][2] - outs[1][2]).abs().max() < 3e-2


def test_droid_frontend_end_to_end():
    """MotionFilter + DroidFrontend (the reference's own driver loop) on the procedural stream"""
    from nerf_slam_b200.droid import DepthVideo, DroidFrontend, MotionFilter
    from nerf_slam_b200.synthetic import SyntheticRoom
    H, W = 240, 320
    net = _net()
    room = SyntheticRoom(W, H, 60, seed=0, step=0.03)
    video = DepthVideo((H, W), buffer=64, device=DEV)
    args = types.SimpleNamespace(warmup=8, beta=0.3, frontend_nms=1, keyframe_thresh=4.0, frontend_window=25,
                                 frontend_thresh=16.0, frontend_radius=2, upsample=True)
    filt = MotionFilter(net, video, min_flow_thresh=2.4, device=DEV)
    front = DroidFrontend(net, video, args)
    gt = []
    for k in range(60):
        p = room.packet(k)
        img = torch.as_tensor(np.asarray(p["images"]))[..., [2, 1, 0]].permute(0, 3, 1, 2).contiguous()
        n0 = video.counter.value
        filt.track(k, float(p["t_cams"][0]), img, None, torch.as_tensor(p["calibs"][0].camera_model.numpy()))
        if video.counter.value > n0:
            gt.append((video.counter.value - 1, np.asarray(p["poses"][0], np.float64)))
        front()
    torch.cuda.synchronize()
    assert front.is_initialized
    n = front.t1
    g = front.graph
    assert len(g.ii) <= g.max_factors + 2 and len(set(zip(g.ii.tolist(), g.jj.tolist()))) == len(g.ii)
    assert len(g.correlation_volumes) == len(g.ii)
    assert torch.isfinite(video.poses[:n]).all() and (video.disps[:n] >= 1e-3).all()
    assert torch.allclose(video.poses[:n, 3:].norm(dim=-1), torch.ones(n, device=DEV), atol=1e-4)
    assert video.dirty[:n].any() and video.ready.value == 1
