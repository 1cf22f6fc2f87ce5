"""The per-frame palette warp (blinky_warp_device_view_rgba_tables) is GPU-only: a host-only context refuses it before
it looks at any argument, and launches nothing.  The Python binding refuses tables that are not a CUDA tensor before
it calls the library."""
import numpy as np
import pytest


@pytest.fixture()
def built_host(host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.build_lensmap(64, 48, 32)
    return host


def test_host_only_context_refuses_the_tables_warp(bb, built_host):
    host = built_host
    for tables, stride in ((0, 0), (0x1000, 1024)):
        rc = host._lib.blinky_warp_device_view_rgba_tables(host._ctx, 0, 6 * 32 * 32, 0, 56 * 80 * 4, 80 * 4, 4, 2, 2, 1,
                                                           tables, stride, None)
        assert rc == bb.E_NODEVICE
        assert "no CPU fallback" in host._lib.blinky_last_error(host._ctx).decode()
    assert host.launch_count == 0


def test_tables_must_be_a_cuda_tensor(bb, built_host):
    import torch

    host = built_host
    for tables in (np.zeros((2, 256), np.uint32), torch.zeros((2, 256), dtype=torch.int32), [0] * 256):
        with pytest.raises(ValueError):
            host.warp_view(0, 0, x0=4, y0=2, rowbytes=80 * 4, nframes=2, rgba=True, tables=tables)
        with pytest.raises(ValueError):
            host.warp(0, 0, nframes=2, rgba=True, tables=tables)
    assert host.launch_count == 0
