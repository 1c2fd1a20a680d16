"""CPU: the C-ABI library loads, exports every symbol include/*.h declares, and refuses to run without a GPU."""
import ctypes
import os
import re

import pytest

import opencv_b200 as cvb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = []
    for h in ("b200cv.h", "b200cv_hal.h", "b200cv_batch.h"):
        txt = open(os.path.join(ROOT, "include", h)).read()
        txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
        names += re.findall(r"B200CV_API\s+[\w\s\*]+?\b(b200cv_\w+)\s*\(", txt)
    return sorted(set(names))


def test_library_exports_every_declared_symbol():
    L = cvb.lib()
    names = declared_symbols()
    assert len(names) > 60
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, "declared in include/*.h but not exported: %s" % missing


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = cvb.lib()
    assert L.b200cv_device_count() == 0
    rc = L.b200cv_init(0)
    assert rc == -4, "b200cv_init must fail loudly without a device"
    assert b"no CPU fallback" in L.b200cv_last_error()
    with pytest.raises(cvb.B200cvError):
        cvb.init(0)


def test_host_tables_are_pure_host_code():
    # these exported helpers run on the CPU by design (coefficient tables), no device needed
    k = cvb.getGaussianKernelFixed8(5, 0)
    assert list(k) == [16, 64, 96, 64, 16]
    assert abs(cvb.getGaussianKernel(7, 1.5).sum() - 1) < 1e-12


def test_cpp_host_mirror_compiles_against_the_c_abi():
    """the C++ mirror (cv:: signatures, Stream/Event/GpuMat/Filter) builds with plain g++ against include/*.h + the shared library"""
    import subprocess
    src = os.path.join(ROOT, "tests", "cpp", "test_host_api.cpp")
    exe = os.path.join(ROOT, "tests", "cpp", "test_host_api")
    lib = os.path.join(ROOT, "opencv_b200", "lib")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-o", exe, src, "-L" + lib, "-lb200cv", "-Wl,-rpath,$ORIGIN/../../opencv_b200/lib"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    import torch
    if not torch.cuda.is_available():
        run = subprocess.run([exe], capture_output=True, text=True)
        assert run.returncode == 1 and "no CPU fallback" in run.stderr      # loud failure without a device


def test_cv_typed_surface_compiles_against_the_reference_headers():
    """b200cv_opencv.hpp (cv::InputArray / OutputArray / cv::cuda::GpuMat / HostMem) builds against the reference's headers and links with
    the reference's core + imgproc; without a device the binary fails loudly"""
    import subprocess
    from oracle import build_cv_surface
    if not os.path.isdir(os.path.join(build_cv_surface.REF, "modules", "core", "include")) or not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libocvref.so")):
        pytest.skip("needs the reference's sources and oracle/_ref")
    exe = build_cv_surface.build()
    assert exe and os.path.exists(exe)
    import torch
    if not torch.cuda.is_available():
        run = subprocess.run([exe], capture_output=True, text=True)
        assert run.returncode == 1 and "no CPU fallback" in run.stderr
