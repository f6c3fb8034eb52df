"""CPU: the reciprocal of the reprojection kernel (rp_rcp in psm_reproject.cuh), compiled for the host, against IEEE
1.0 / h bit for bit: random bit patterns, every exponent with edge and random mantissas, powers of two and the values
next to them, and the overflow / underflow edges.  The device build differs only in its float seed, which the exact
remainder correction makes irrelevant to the result."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

DRIVER = r"""
#include "%s"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
static unsigned long long bits(double x) { unsigned long long u; std::memcpy(&u, &x, 8); return u; }
static double dbl(unsigned long long u) { double x; std::memcpy(&x, &u, 8); return x; }
int main()
{
    std::mt19937_64 g(7);
    long bad = 0, n = 0;
    auto chk = [&](double h) {
        const double a = psm::rp_rcp(h), b = 1.0 / h;
        ++n;
        if (!(bits(a) == bits(b) || (a != a && b != b))) { if (bad < 5) std::printf("h=%%a got %%a want %%a\n", h, a, b); ++bad; }
    };
    for (long i = 0; i < 2000000; ++i) chk(dbl(g()));
    const unsigned long long edge[4] = {0, 1, 0xfffffffffffffull, 0xffffffffffffeull};
    for (unsigned long long e = 0; e < 2048; ++e)
        for (int k = 0; k < 400; ++k) {
            const unsigned long long m = k < 4 ? edge[k] : (k < 40 ? g() >> (12 + k %% 52) : g() & 0xfffffffffffffull);
            chk(dbl(e << 52 | m));
            chk(-dbl(e << 52 | m));
        }
    for (int k = -1074; k <= 1023; ++k) { chk(std::ldexp(1.0, k)); chk(std::ldexp(3.0, k)); chk(std::nextafter(std::ldexp(1.0, k), 0.0)); }
    chk(5.562684646268003e-309); chk(5.562684646268004e-309); chk(0.0); chk(-0.0); chk(INFINITY); chk(-INFINITY); chk(NAN);
    std::printf("%%ld checked, %%ld differ\n", n, bad);
    return bad != 0;
}
"""


def test_reciprocal_equals_ieee_division(tmp_path):
    if not shutil.which(NVCC) and not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    src = tmp_path / "rcp.cu"
    src.write_text(DRIVER % os.path.join(ROOT, "primestereomatch_b200", "csrc", "psm_reproject.cuh"))
    exe = tmp_path / "rcp"
    subprocess.run([NVCC, "-O2", "-std=c++17", "-Xcompiler", "-ffp-contract=off", "-o", str(exe), str(src)], check=True,
                   capture_output=True, timeout=600)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout
    assert " 0 differ" in out.stdout
