"""harness/room.py: the cfg5 scene the scene-layout benchmarks are measured on stays the same scene bit for bit."""
import hashlib

from harness import room

# sha256 over build_scene("cpu") (every group's leaves in order) and scene_camera(k, 512) for k < 8, as
# benchmarks/scene_step.py built them when the scene lived there
CFG5_SHA256 = "5b1ecf5024d48b98426665fd3ae5ab96c9705bb9a98fd60d4d2587cc6f1e1a15"


def test_cfg5_scene_and_cameras_are_bit_identical():
    h = hashlib.sha256()
    for g in room.build_scene("cpu"):
        for k, v in g.items():
            h.update(k.encode())
            h.update(v.detach().numpy().tobytes())
    for k in range(8):
        c = room.scene_camera(k, 512, "cpu")
        for t in (c.world_view_transform, c.full_proj_transform, c.camera_center):
            h.update(t.numpy().tobytes())
    assert h.hexdigest() == CFG5_SHA256


def test_small_room_inputs_are_activated_and_sized():
    sc = room.rasterizer_inputs(room.build_scene("cpu", n_wall=100, n_floor=50, n_obj=20, scale_mul=4.0))
    assert sc["means3D"].shape == (5 * 100 + 50 + 4 * 20, 3) and sc["shs"].shape[1:] == (4, 3)
    assert float(sc["opacities"].min()) > 0 and float(sc["opacities"].max()) < 1
    assert float((sc["rotations"].norm(dim=1) - 1).abs().max()) < 1e-6
