"""CONV_KERNELS of test_conv_calls_fp64_gpu.py is exactly the set of convolution kernel instantiations compiled into
libscsfm.so (the kernel symbols of its sm_90a cubin, demangled), so the list the coverage test checks cannot go stale when
a kernel template gains or loses an instantiation.  Skips where cuobjdump is not installed."""
import os
import re
import shutil
import subprocess

import pytest

from test_conv_calls_fp64_gpu import CONV_FAMILY, CONV_KERNELS, kernel_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sc-sfmlearner-release_b200", "scsfm", "libscsfm.so")


def _tool(name):
    path = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return shutil.which(name) or (path if os.path.exists(path) else None)


def test_conv_kernel_list_matches_library():
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not installed")
    demangler = _tool("c++filt") or _tool("cu++filt")
    assert demangler is not None, "neither c++filt nor cu++filt found next to cuobjdump"
    if not os.path.exists(LIB):
        subprocess.check_call([os.path.join(ROOT, "sc-sfmlearner-release_b200", "build.sh")])
    elf = subprocess.run([cuobjdump, "-elf", LIB], capture_output=True, text=True, check=True).stdout
    mangled = sorted(set(re.findall(r"\.text\.(_ZN5scsfm\w+)", elf)))
    assert mangled, "no scsfm kernels in the cubin of %s" % LIB
    names = subprocess.run([demangler], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout
    built = {kernel_key(n) for n in names.splitlines() if n.strip()}
    conv = {k for k in built if CONV_FAMILY.match(k)}
    assert len(CONV_KERNELS) == len(set(CONV_KERNELS)) == 56
    assert conv == set(CONV_KERNELS), ("in the library only: %s; listed only: %s" % (sorted(conv - set(CONV_KERNELS)),
                                                                                     sorted(set(CONV_KERNELS) - conv)))
