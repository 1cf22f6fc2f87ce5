"""The C-ABI library loads and exports every symbol include/blinky_b200.h declares;
GPU entry points fail loudly on a host-only context (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "blinky_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(blinky_[a-z0-9_]+)\s*\(", src)) - {"blinky_print_fn", "blinky_exec_fn"})


def test_header_and_binding_agree(bb):
    assert declared_symbols() == sorted(bb.EXPORTED_SYMBOLS)


def test_every_declared_symbol_is_exported(bb):
    lib = ctypes.CDLL(bb.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), name


def test_library_is_in_tree_and_native(bb):
    assert os.path.dirname(bb.LIB_PATH) == os.path.join(ROOT, "blinky_b200")
    data = open(bb.LIB_PATH, "rb").read()
    assert data[:4] == b"\x7fELF"
    # the kernels are really in there, compiled for sm_90a
    assert b"warp_gather_kernel" in data and b"sm_90a" in data


def test_host_only_context_refuses_the_hot_path(bb, host):
    host.command("f_globe cube")
    host.command("f_lens panini")
    host.build_lensmap(64, 48, 32)
    faces = bb.synthetic_faces(6, 32)
    with pytest.raises(bb.BlinkyError) as e:
        host.warp_host(faces.reshape(1, -1))
    assert e.value.code == bb.E_NODEVICE and "no CPU fallback" in str(e.value)
    with pytest.raises(bb.BlinkyError) as e:
        host.warp(0, 0)
    assert e.value.code == bb.E_NODEVICE
    with pytest.raises(bb.BlinkyError):
        host.set_background(None)
    assert host.launch_count == 0


def test_missing_library_is_loud(bb, monkeypatch, tmp_path):
    import importlib

    monkeypatch.setattr(bb, "LIB_PATH", str(tmp_path / "nope.so"))
    monkeypatch.setattr(bb, "_lib", None)
    with pytest.raises(ImportError) as e:
        bb.load_library()
    assert "no CPU fallback" in str(e.value)


def test_error_codes_and_messages(bb, host):
    with pytest.raises(bb.BlinkyError) as e:
        host.command("f_nonsense 1")
    assert e.value.code == bb.E_INVALID
    with pytest.raises(bb.BlinkyError) as e:
        host.load_lens("does_not_exist")
    assert e.value.code == bb.E_SCRIPT
    assert "could not loadfile" in host.log and "not a valid lens" in host.log
    with pytest.raises(bb.BlinkyError) as e:
        host.build_lensmap(64, 48, 32)
    assert e.value.code == bb.E_STATE
    with pytest.raises(bb.BlinkyError) as e:
        host.build_lensmap(0, 48, 32)
    assert e.value.code == bb.E_INVALID
    with pytest.raises(bb.BlinkyError):
        host.lensmap_packed() if False else host.set_zoom(99)
    assert bb.load_library().blinky_version().startswith(b"blinky_b200")


def test_c_example_builds_links_and_refuses_to_warp_without_a_gpu(bb, tmp_path):
    """examples/headless_warp.c against include/blinky_b200.h + the in-tree .so, as a C host would"""
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "headless_warp")
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    r = subprocess.run(["gcc", "-O2", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "headless_warp.c"),
                        "-L", os.path.dirname(bb.LIB_PATH), "-lblinky_b200", "-Wl,-rpath," + os.path.dirname(bb.LIB_PATH), "-o", exe],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[:2000]
    r = subprocess.run([exe, "-1", "hammer", "320", "200", "96", "2"], capture_output=True, text=True, cwd=root)
    assert r.returncode == 3, (r.returncode, r.stdout, r.stderr)  # BLINKY_E_NODEVICE path
    assert "40176 mapped pixels" in r.stdout and "f_lens hammer; f_contain" in r.stdout
    assert "no CPU fallback" in r.stderr
