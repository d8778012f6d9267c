"""The resolve rule C17 (DESIGN.md §4) in its numpy restatement (oracle/resolve.py), checked by hand, against the oracle's
C11 RGBA, and the CLIs' --supersample refusals, which happen before any device is touched."""
import numpy as np
import pytest

from oracle import render
from oracle import resolve as R

FORMATS = ("rgba", "rgb", "rgb_planar", "gray")


def _playpal(seed):
    return np.random.default_rng(seed).integers(0, 256, (256, 3), dtype=np.uint8)


def test_factor_one_rgba_is_the_oracle_c11_rgba(oracle_scene, synth_wad):
    from oracle import wad as W
    from rust_doom_b200 import poses as P
    import rust_doom_b200 as b2d
    pal = W.TextureDirectory(W.Archive(synth_wad)).palettes[0]
    scene = b2d.Scene(b2d.Archive.from_bytes(synth_wad), 0)
    poses = np.concatenate([scene.start_pose, P.flythrough_poses(scene, 3, 2)])
    idx, rgba = render.render(oracle_scene, render.make_view(96, 60), poses, rgba=True)
    assert np.array_equal(R.resolve(idx, [pal], 1, "rgba"), rgba)
    assert np.array_equal(R.resolve(idx, [pal], 1, "rgb"), rgba.view(np.uint8).reshape(len(poses), 60, 96, 4)[..., :3])


@pytest.mark.parametrize("k", range(1, 9))
def test_uniform_block_gives_its_palette_colour(k):
    pal = _playpal(k)
    idx = np.full((2, 2 * k, 3 * k), 7, np.uint8)
    idx[1] = 200
    r, g, b = (int(v) for v in pal[7])
    out = R.resolve(idx, [pal], k, "rgb")
    assert out.shape == (2, 2, 3, 3) and (out[0] == pal[7]).all() and (out[1] == pal[200]).all()
    assert (R.resolve(idx, [pal], k, "rgba")[0] == (r | g << 8 | b << 16 | 0xFF000000)).all()
    assert (R.resolve(idx, [pal], k, "rgb_planar")[0] == pal[7][:, None, None]).all()
    assert (R.resolve(idx, [pal], k, "gray")[0] == (77 * r + 150 * g + 29 * b + 128) >> 8).all()


def test_half_up_rounding_by_hand():
    """2 x 2 blocks whose red sums are 1, 2, 3, 6 (means 0.25, 0.5, 0.75, 1.5) and 3 x 3 blocks with sums 4, 5, 13, 14
    (means 0.44, 0.56, 1.44, 1.56): (sum + k*k // 2) // (k*k) rounds halves up."""
    pal = np.zeros((256, 3), np.uint8)
    pal[1] = (1, 0, 0)
    pal[2] = (2, 0, 0)
    blocks2 = [[[1, 0], [0, 0]], [[1, 1], [0, 0]], [[1, 1], [1, 0]], [[2, 2], [1, 1]]]
    idx = np.concatenate([np.array(b, np.uint8) for b in blocks2], axis=1)[None]          # 1 frame, 2 x 8
    assert R.resolve(idx, [pal], 2, "rgb")[0, 0, :, 0].tolist() == [0, 1, 1, 2]
    blocks3 = [[1, 1, 1, 1, 0, 0, 0, 0, 0], [1] * 5 + [0] * 4, [2] * 4 + [1] * 5, [2] * 5 + [1] * 4]
    idx = np.concatenate([np.array(b, np.uint8).reshape(3, 3) for b in blocks3], axis=1)[None]
    assert R.resolve(idx, [pal], 3, "rgb")[0, 0, :, 0].tolist() == [0, 1, 1, 2]
    # green and blue are averaged the same way, each channel on its own
    pal[3] = (0, 255, 1)
    idx = np.array([[[3, 0], [0, 0]]], np.uint8)
    assert R.resolve(idx, [pal], 2, "rgb")[0, 0, 0].tolist() == [0, 64, 0]          # 255/4 = 63.75; 1/4 = 0.25


def test_luma_table_by_hand():
    pal = np.zeros((256, 3), np.uint8)
    pal[1], pal[2], pal[3] = (255, 0, 0), (0, 255, 0), (200, 100, 50)
    y = R.luma(pal)
    assert y[1] == 77          # (77 * 255 + 128) >> 8 = 19763 >> 8
    assert y[2] == 149         # (150 * 255 + 128) >> 8 = 38378 >> 8
    assert y[3] == 124         # (15400 + 15000 + 1450 + 128) >> 8 = 31978 >> 8
    assert y[0] == 0 and R.luma(np.full((256, 3), 255, np.uint8))[0] == 255
    idx = np.array([[[1, 2], [3, 0]]], np.uint8)
    assert R.resolve(idx, [pal], 2, "gray")[0, 0, 0] == (77 + 149 + 124 + 0 + 2) // 4


def test_levels_pick_each_frames_palette_and_formats_agree():
    pals = [_playpal(1), 255 - _playpal(1)]
    rng = np.random.default_rng(5)
    idx = rng.integers(0, 256, (4, 12, 18), dtype=np.uint8)
    lv = [0, 1, 1, 0]
    for k in (1, 2, 3, 6):
        rgb = R.resolve(idx, pals, k, "rgb", lv)
        for f in range(4):
            assert np.array_equal(rgb[f], R.resolve(idx[f:f + 1], [pals[lv[f]]], k, "rgb")[0])
        assert np.array_equal(R.resolve(idx, pals, k, "rgb_planar", lv), rgb.transpose(0, 3, 1, 2))
        packed = R.resolve(idx, pals, k, "rgba", lv)
        assert np.array_equal(packed.view(np.uint8).reshape(rgb.shape[:3] + (4,))[..., :3], rgb)
    assert np.array_equal(R.resolve(idx, pals, 2, "rgb"), R.resolve(idx, pals, 2, "rgb", [0] * 4))


@pytest.mark.parametrize("argv", [["--supersample", "0"], ["--supersample", "9"],
                                  ["--supersample", "2", "--levels", "0", "--world", "2", "--id-file", "x"]])
def test_cli_refuses_bad_supersample(argv, capsys):
    from rust_doom_b200 import cli
    assert cli.main(["--resolution", "160x100"] + argv) == 2
    assert "--supersample" in capsys.readouterr().err


@pytest.mark.parametrize("res,k", [("2049x100", 2), ("1920x1080", 3), ("640x1081", 2)])
def test_cli_refuses_supersampled_size_past_the_view_limits(b2d, res, k, capsys):
    """K*W past 4096 or K*H past 2160 is the view's own error, raised before a renderer (and a device) is asked for."""
    from rust_doom_b200 import cli
    assert cli.main(["--resolution", res, "--supersample", str(k)]) == 1
    err = capsys.readouterr().err
    assert "view out of range" in err and "CUDA" not in err
    assert cli.main(["--resolution", res, "--supersample", str(k), "--levels", "0"]) == 1
    assert "view out of range" in capsys.readouterr().err


def test_compiled_cli_refuses_bad_supersample(tmp_path):
    import subprocess
    from rust_doom_b200 import synthwad
    from tests.test_cli import _b2d_binary
    wad = tmp_path / "syn.wad"
    wad.write_bytes(synthwad.build_iwad(1, ("E1M1",)))
    exe = _b2d_binary()
    for k in ("0", "9"):
        out = subprocess.run([exe, "-i", str(wad), "-r", "160x100", "--supersample", k], capture_output=True, text=True)
        assert out.returncode == 2 and "--supersample" in out.stderr
    out = subprocess.run([exe, "-i", str(wad), "-r", "2049x100", "--supersample", "2"], capture_output=True, text=True)
    assert out.returncode == 1 and "view out of range" in out.stderr
