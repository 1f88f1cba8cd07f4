"""The C-ABI library loads on a CPU-only box, exports every symbol the headers declare, and the
CUDA engine fails loudly (no CPU fallback) when there is no device."""
import ctypes
import os
import re

import pytest

from agentcontrolplane_b200 import _lib
from agentcontrolplane_b200.engine import Engine, EngineError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(acp_[a-z_0-9]+)\s*\(", text)))


@pytest.mark.parametrize("header", ["acp_infer.h", "acp_infer_kernels.h", "acp_host.h"])
def test_every_declared_symbol_is_exported(header):
    lib = _lib.load_host() if header == "acp_host.h" else _lib.load()
    names = _declared(header)
    assert names, header
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/{header} but not exported"


def test_expected_boundary_entry_points_present():
    assert set(_declared("acp_infer.h")) >= {
        "acp_infer_init", "acp_infer_submit", "acp_infer_wait", "acp_infer_poll", "acp_infer_result",
        "acp_infer_cancel", "acp_infer_stats", "acp_infer_free", "acp_infer_shutdown"}


def test_version_and_no_device_behaviour():
    lib = _lib.load()
    lib.acp_infer_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.acp_infer_version()
    if lib.acp_kernel_device_count() == 0:
        with pytest.raises(EngineError) as ei:
            Engine({"model": "tiny"})
        assert ei.value.code == -5          # ACP_ERR_CUDA: loud failure, never a CPU path


def test_default_kernel_dispatch():
    """The kernel the GEMM dispatcher picks by default, with no environment switch set (host logic, no GPU):
    prefill-sized problems (more than 256 rows; bf16, SwiGLU or one fp32 plane) must run the persistent kernel,
    everything else the tiled one — an inverted default here silently slows every prefill step."""
    import subprocess, sys
    code = (
        "import os\n"
        "os.environ.pop('ACP_GEMM_PERSISTENT', None)\n"
        "from agentcontrolplane_b200 import _lib\n"
        "p = _lib.load().acp_kernel_gemm_path\n"
        "print(p(28672, 4096, 4096, 1, 3, 0), p(4096, 8192, 14336, 1, 0, 0), p(4096, 64, 4096, 1, 0, 0), p(4096, 256, 4096, 1, 0, 0),\n"
        "      p(4096, 512, 4096, 2, 1, 0), p(8192, 4096, 1024, 1, 1, 0), p(4224, 4096, 4096, 1, 0, 0),\n"
        "      p(4096, 4096, 4096, 1, 0, -1), p(4096, 4096, 4096, 1, 0, 256), p(4096, 4096, 4096, 1, 2, 0))\n")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    #          gate/up  down  decode  N=256  2 fp32 planes  1 fp32 plane (TP prefill)  odd m-tiles  forced persistent  forced tile  arg-max
    assert out.stdout.split() == ["1", "1", "0", "0", "0", "1", "1", "1", "0", "0"], out.stdout


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "agentcontrolplane_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cc", ".cu", ".h", ".cuh")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_host_library_is_independent_of_the_product():
    """libacp_host.so (the reference-side mirror + CPU baseline) neither links nor needs libacp_infer.so
    or CUDA: bench.py --impl reference maps it alone."""
    import subprocess
    out = subprocess.run(["ldd", _lib.HOST_LIB_PATH], capture_output=True, text=True).stdout
    assert "libacp_infer" not in out and "libcuda" not in out and "libcudart" not in out, out
    nm = subprocess.run(["nm", "-D", "--undefined-only", _lib.HOST_LIB_PATH], capture_output=True, text=True).stdout
    assert "acp_infer_" not in nm and "cuda" not in nm.lower(), nm
    code = ("import ctypes, json, sys; sys.path.insert(0, %r)\n"
            "from agentcontrolplane_b200 import host\n"
            "with host.StubServer() as srv:\n"
            "    r = host.hostsim_run({'tasks': 20, 'workers': 2, 'provider': 'openai', 'model': 'gpt-4o', 'baseURL': srv.base_url})\n"
            "maps = open('/proc/self/maps').read()\n"
            "assert 'libacp_host.so' in maps and 'libacp_infer' not in maps and 'libcuda' not in maps, maps\n"
            "print(r['reconciles'])") % ROOT
    res = subprocess.run([__import__("sys").executable, "-c", code], capture_output=True, text=True)
    assert res.returncode == 0 and res.stdout.strip() == "20", res.stderr
