"""Several images per run, host side: command-line expansion and the per-image output layout, per-object random draws against
single runs seeded the same way, and the batched background-removal host steps against U2netSession.predict."""
import argparse

import numpy as np
import pytest
import torch

import pipeline_i2v_eval_v01 as P1
import pipeline_i2v_eval_v02 as P2
from hi3d_official_b200 import engine, rembg


def parse(stage, *argv):
    ap = argparse.ArgumentParser()
    P1.add_cli_args(ap, stage)
    return ap.parse_args(list(argv))


@pytest.mark.parametrize("stage", [1, 2])
def test_defaults_are_one_image(stage):
    p = parse(stage)
    assert p.image_path == ["demo/15_out.png"] and p.elevation == [0] and p.seed is None and p.towers is None
    assert p.batch == 1 and p.output_dir == "outputs/15_out"
    assert p.denoise_config == f"configs/inference-v0{stage}.yaml"


def test_per_image_expansion():
    assert P1.per_image(None, 3, "--seed") == [None] * 3
    assert P1.per_image([7], 3, "--seed") == [7, 7, 7]
    assert P1.per_image([1, 2, 3], 3, "--seed") == [1, 2, 3]
    with pytest.raises(SystemExit):
        P1.per_image([1, 2], 3, "--seed")


def test_batch_plan_layout():
    p = parse(1, "--image_path", "in/a.png", "x/b.jpg", "c.png", "--output_dir", "out", "--seed", "1", "2", "3",
              "--elevation", "10", "--towers", "t.pt", "--batch", "2")
    plan = P1.batch_plan(p)
    assert plan["dirs"] == ["out/a", "out/b", "out/c"]
    assert plan["seeds"] == [1, 2, 3] and plan["elevations"] == [10] * 3 and plan["towers"] == ["t.pt"] * 3
    assert plan["groups"] == [[0, 1], [2]]
    assert P1.batch_plan(parse(1, "--image_path", "a.png", "b.png", "--batch", "5"))["groups"] == [[0, 1]]
    seeds = P1.batch_plan(parse(2, "--image_path", "a.png", "b.png"))["seeds"]
    assert len(seeds) == 2 and all(0 <= s <= 65535 for s in seeds)


@pytest.mark.parametrize("argv", [["--image_path", "a/x.png", "b/x.png"], ["--image_path", "a.png", "b.png", "--batch", "0"],
                                  ["--image_path", "a.png", "b.png", "--cond", "c.pt"],
                                  ["--image_path", "a.png", "b.png", "c.png", "--seed", "1", "2"]])
def test_batch_plan_rejects(argv):
    with pytest.raises(SystemExit):
        P1.batch_plan(parse(1, *argv))


def test_load_towers_stacks_per_key(tmp_path):
    paths = []
    for i in range(2):
        paths.append(str(tmp_path / f"t{i}.pt"))
        torch.save({"clip": torch.full((1, 1024), float(i)), "aes": torch.tensor([[5.0 + i]]),
                    "depth": torch.full((16, 24, 24), float(i))}, paths[-1])
    t = P1.load_towers(paths)
    assert t["clip"].shape == (2, 1024) and t["aes"].shape == (2, 1) and t["depth"].shape == (32, 24, 24)
    assert float(t["aes"][1, 0]) == 6.0 and float(t["depth"][16:].min()) == 1.0 and float(t["clip"][0].max()) == 0.0


def test_cat_cond_is_object_major():
    ds = [dict(crossattn=torch.full((1, 1, 4), float(i)), concat=torch.full((3, 2, 1, 1), float(i))) for i in range(2)]
    c = P1.cat_cond(ds)
    assert c["crossattn"][:, 0, 0].tolist() == [0.0, 1.0] and c["concat"][:, 0, 0, 0].tolist() == [0, 0, 0, 1, 1, 1]


# ---- random numbers ------------------------------------------------------------------------------------------------------------
def test_per_object_draws_match_single_runs():
    """Each object draws the condition-frame noise, then the initial latents, from its own generator: the numbers a run that
    seeded the global generator with the object's seed draws in the same order."""
    seeds, T = [3, 11, 3], 4
    video = torch.zeros(len(seeds), 3, T, 8, 8)
    gens = [torch.Generator().manual_seed(s) for s in seeds]
    noise = engine.randn_like_per_object([video[b:b + 1, :, 0] for b in range(len(seeds))], gens)
    lat = engine.per_object_randn((T, 4, 2, 2), gens, "cpu")
    assert noise.shape == (len(seeds), 3, 8, 8) and lat.shape == (len(seeds) * T, 4, 2, 2)
    for i, s in enumerate(seeds):
        with torch.random.fork_rng():
            torch.manual_seed(s)
            n1 = torch.randn_like(video[i:i + 1, :, 0])
            l1 = torch.randn(T, 4, 2, 2)
        assert torch.equal(noise[i:i + 1], n1) and torch.equal(lat[i * T:(i + 1) * T], l1)
    assert torch.equal(noise[0], noise[2]) and not torch.equal(noise[0], noise[1])


def test_per_object_noise_keeps_the_layout_of_a_view():
    """Stage 2 draws the condition-frame noise like a (T, 3, H, W) permuted VIEW of one clip; several clips make a contiguous
    copy.  Per object the draws must follow the view's memory order, as the single run's randn_like does."""
    seeds, T = [2, 8], 4
    video = torch.zeros(len(seeds), 3, T, 5, 5)
    frames_of = lambda v: v.permute(0, 2, 1, 3, 4).reshape(-1, 3, 5, 5)     # noqa: E731
    assert not frames_of(video[:1]).is_contiguous() and frames_of(video).is_contiguous()
    noise = engine.randn_like_per_object([frames_of(video[b:b + 1]) for b in range(2)],
                                         [torch.Generator().manual_seed(s) for s in seeds])
    for i, s in enumerate(seeds):
        with torch.random.fork_rng():
            torch.manual_seed(s)
            ref = torch.randn_like(frames_of(video[i:i + 1]))
            torch.manual_seed(s)
            contiguous = torch.randn(T, 3, 5, 5)
        assert torch.equal(noise[i * T:(i + 1) * T], ref) and not torch.equal(ref, contiguous)


@pytest.mark.parametrize("chunk", [1, 16, None])
def test_posterior_noise_matches_the_encode_draws(chunk):
    """The stage-2 encode of a single run draws CPU randn once per chunk of en_and_decode_n_samples_a_time frames."""
    T, h, seeds = 16, 2, [5, 9]
    model = argparse.Namespace(en_and_decode_n_samples_a_time=chunk)
    got = P2.posterior_noise(model, T, h, [torch.Generator().manual_seed(s) for s in seeds])
    k = chunk or T
    for i, s in enumerate(seeds):
        with torch.random.fork_rng():
            torch.manual_seed(s)
            ref = torch.cat([torch.randn((min(k, T - t), 4, h, h)) for t in range(0, T, k)], 0)
        assert torch.equal(got[i * T:(i + 1) * T], ref)


def test_per_object_noise_needs_one_generator_per_object():
    with pytest.raises(ValueError):
        engine.randn_like_per_object([torch.zeros(2, 3)] * 3, [torch.Generator()] * 2)


# ---- background removal ----------------------------------------------------------------------------------------------------------
class _StubNet:
    """Per-image stand-in for U^2-Net: a smooth function of each image alone; records the batch sizes it saw."""

    def __init__(self):
        self.calls = []

    def __call__(self, x):
        self.calls.append(tuple(x.shape))
        return torch.sigmoid(x.mean(1) * 1.7 + x[:, 0] * x[:, 2])


def _images():
    from PIL import Image
    rs = np.random.RandomState(0)
    return [Image.fromarray((rs.rand(hh, ww, 3) * 255).astype("uint8")) for hh, ww in ((200, 160), (90, 300), (320, 320))]


def test_batched_rembg_host_steps_match_predict():
    imgs = _images()
    net = _StubNet()
    masks = rembg.U2netSession(net).predict_batch(imgs)
    assert net.calls == [(3, 3, 320, 320)]
    single = rembg.U2netSession(_StubNet())
    for img, m in zip(imgs, masks):
        ref = single.predict(img)
        assert m.size == img.size and m.mode == "L"
        assert np.array_equal(np.asarray(m), np.asarray(ref))


def test_remove_batch_matches_remove():
    imgs = _images()
    session = rembg.U2netSession(_StubNet())
    for img, cut in zip(imgs, rembg.remove_batch(imgs, session)):
        ref = rembg.remove(img, session)
        assert cut.mode == ref.mode == "RGBA" and cut.size == img.size
        assert np.array_equal(np.asarray(cut), np.asarray(ref))
