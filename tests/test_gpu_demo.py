"""The reference's pipeline on hardware (SURVEY.md §8f-1/2/3): DataModule -> SlamModule(VioSLAM) -> FusionModule wired
and spun exactly as the reference's examples/slam_demo.py does in sequential mode (:160-181), through the import-path
shim, on the procedural stream written to disk in the reference's dataset format — with the NeRF trainer and with the
Sigma-fusion volume as consumers."""
import os
import sys
import types
from queue import Queue

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "nerf_slam_b200", "shim")
WEIGHTS = os.path.join(ROOT, "oracle", "_ref", "droid.pth")


def _args(dataset_dir, fusion, buffer=24):
    return types.SimpleNamespace(parallel_run=False, multi_gpu=False, initial_k=0, final_k=-1, img_stride=1, stereo=False,
                                 weights=WEIGHTS if os.path.exists(WEIGHTS) else None, buffer=buffer, dataset_dir=str(dataset_dir),
                                 dataset_name="nerf", mask_type="ours", slam=True, fusion=fusion, gui=False, width=0, height=0,
                                 network="", eval=False, tsdf_resolution=192)


@pytest.mark.parametrize("fusion", ["nerf", "sigma"])
def test_reference_pipeline_wiring_and_fusion_volume_on_hardware(tmp_path, monkeypatch, fusion):
    from nerf_slam_b200 import datasets, synthetic
    room = synthetic.SyntheticRoom(320, 240, 56, seed=0, step=0.03)
    datasets.write_transforms_dataset(room, str(tmp_path))
    monkeypatch.setattr(sys, "path", [SHIM, ROOT] + [p for p in sys.path if p not in (SHIM, ROOT)])
    for m in [k for k in sys.modules if k.split(".")[0] in ("datasets", "slam", "fusion", "pipeline", "gui")]:
        monkeypatch.delitem(sys.modules, m)
    from datasets.data_module import DataModule               # the reference's import paths, resolved by the shim
    from fusion.fusion_module import FusionModule
    from slam.slam_module import SlamModule
    args = _args(tmp_path, fusion)
    args.world_T_imu_t0 = np.linalg.inv(np.asarray(room.packet(0)["poses"][0]))
    data_q, slam_q = Queue(), Queue()
    data = DataModule(args.dataset_name, args, device="cpu")
    slam = SlamModule("VioSLAM", args, device="cuda:0")
    fus = FusionModule(args.fusion, args, device="cuda:0")
    data.register_output_queue(data_q); slam.register_input_queue("data", data_q)
    slam.register_output_queue(slam_q); fus.register_input_queue("slam", slam_q)
    steps = 0
    while data.spin() and slam.spin() and fus.spin():         # examples/slam_demo.py:171-175
        steps += 1
        assert steps < 200
    torch.cuda.synchronize()
    fe = slam.slam.visual_frontend
    assert steps >= 50 and fe.is_initialized and fe.kf_idx >= 9 and fe.ba_failures(wait=True) == 0
    if fusion == "nerf":
        nf = fus.fusion
        # one fit per spin without a new packet (fusion/nerf_fusion.py:237-258: a packet with keyframes is ingested, not fitted)
        assert nf.total_iters >= steps // 2 and nf.ngp.nerf.training.n_images_for_training >= 8
        assert np.isfinite(nf.ngp.sync_stats())
    else:
        vol = fus.fusion
        assert vol.integrated_frames >= 9 and len(vol.history) >= 9
        assert float((vol.volume.weight > 0).float().mean()) > 0.01 and torch.isfinite(vol.volume.tsdf).all()
