"""GroupNorm statistics steps of the launch plans (UNet, VAE encoder, decoder and video decoder): every unit table a
GroupNorm step reads (an apply, or the group sums of a frame-sharded temporal GroupNorm) is written by a statistics step
earlier in the same plan, and every table a statistics step writes is read by a GroupNorm step."""
import pytest

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import configs  # noqa: E402
from hi3d_official_b200.unet import VideoUNet  # noqa: E402
from hi3d_official_b200.vae import AutoencoderKLModeOnly, AutoencoderKLTemporal  # noqa: E402


def _check_tables(steps, name):
    written, read = {}, set()              # id(StatsBuf) -> index of the statistics step that writes it
    for i, s in enumerate(steps):
        for st in getattr(s, "stats_in", ()):
            assert id(st) in written, f"{name}: step {i} reads a table that no earlier statistics step writes"
            read.add(id(st))
        st = getattr(s, "stats_out", None)
        if st is not None:
            written[id(st)] = i
    assert read, f"{name}: no GroupNorm step"
    unread = sorted(i for k, i in written.items() if k not in read)
    assert not unread, f"{name}: statistics steps {unread} write tables that no GroupNorm step reads"


@pytest.mark.parametrize("engine", ["tc5", "mma"])
def test_unet_plan_reads_and_writes_every_table(engine):
    net = VideoUNet(**dict(configs.UNET_STAGE1, model_channels=64)).cuda().half()
    net.set_engine(engine)
    T = 4
    _check_tables(net.get_plan(2 * T, 16, 16, T).steps, f"unet {engine}")


@pytest.mark.parametrize("which,n,hw,T", [("enc", 2, 64, 0), ("dec", 2, 8, 0), ("vdec", 4, 8, 4)])
def test_vae_plans_read_and_write_every_table(which, n, hw, T):
    dd = dict(configs._VAE_DD, ch=64)
    if which == "vdec":
        ae = AutoencoderKLTemporal(embed_dim=4, ddconfig=dd, video_kernel_size=[3, 1, 1], time_mode="conv-only")
    else:
        ae = AutoencoderKLModeOnly(embed_dim=4, ddconfig=dd)
    ae = ae.cuda().half()
    _check_tables(ae._plan(which, n, hw, hw, T).steps, which)
