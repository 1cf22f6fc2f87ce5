"""The view-rectangle warp (blinky_warp_device_view / _rgba) is GPU-only: a host-only context refuses it before it
looks at any argument, and launches nothing."""
import pytest


@pytest.mark.parametrize("rgba", [False, True])
def test_host_only_context_refuses_the_view_warp(bb, host, rgba):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.build_lensmap(64, 48, 32)
    with pytest.raises(bb.BlinkyError) as e:
        host.warp_view(0, 0, x0=4, y0=2, rowbytes=80 * (4 if rgba else 1), nframes=2, keep_unmapped=True, rgba=rgba)
    assert e.value.code == bb.E_NODEVICE and "no CPU fallback" in str(e.value)
    assert host.launch_count == 0
