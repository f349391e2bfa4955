"""The handle's owning buffers (calfkit-sdk_b200/csrc/ck_buf.h), built with g++ against the CUDA runtime on their own.

Without a usable device every allocation fails, which is the path a handle takes when memory runs out: reserve must hand
the error back and leave the buffer empty (no freed pointer, no claimed room), and moving or destroying such buffers must
be safe.  On a device, reserve grows, a reserve that already fits changes nothing, and the keep-prefix form carries the
contents over.  The build goes to a temporary directory keyed by the sources and leaves the tree untouched."""
import hashlib
import os
import subprocess
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "calfkit-sdk_b200", "csrc")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _exe() -> str:
    srcs = [os.path.join(HERE, "ckbuf", "buf_host.cpp"), os.path.join(CSRC, "ck_buf.h")]
    key = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs)).hexdigest()[:16]
    exe = os.path.join(tempfile.gettempdir(), f"ck_buf_host_{os.getuid()}_{key}")
    if not os.path.exists(exe):
        tmp = exe + f".{os.getpid()}"
        lib = os.path.join(CUDA, "lib64")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, "-I", os.path.join(CUDA, "include"),
                               "-o", tmp, srcs[0], "-L", lib, "-lcudart", f"-Wl,-rpath,{lib}"])
        os.replace(tmp, exe)
    return exe


def _run(mode: str) -> str:
    r = subprocess.run([_exe(), mode], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def _has_device() -> bool:
    import torch
    return torch.cuda.is_available()


def test_failed_reserve_leaves_buffer_empty():
    if _has_device():
        pytest.skip("a device is present: allocations succeed")
    out = _run("fail")
    assert out.endswith("ok\n"), out
    assert out.count("reserve failed with cuda") == 2, out      # device and page-locked buffers alike


@pytest.mark.gpu
def test_reserve_grows_and_keeps():
    if not _has_device():
        pytest.skip("no CUDA device")
    assert _run("grow") == "ok\n"
