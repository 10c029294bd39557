"""ctypes front-end of the CPU emulation with thread-block clusters (tests only; see cuda_emu_cluster.h).

A separate build of the kernel-body emulation (build_cluster.sh) that also holds the cluster Four-Step kernels
(csrc/cluster4.cuh).  Its planner sees a cluster-capable device only after set_cluster_capable(True); by default it plans as
the plain emulation does.  Descriptors come from emu.make_desc."""
import ctypes, os, subprocess

import emu

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "_build", "libb200fft_emu_cluster.so")
        srcs = [os.path.join(_HERE, f) for f in ("build_cluster.sh", "emu_cluster_driver.cpp", "emu_cluster_kernels.cpp",
                                                  "emu_driver.cpp", "emu_kernels.cpp", "cuda_emu_cluster.h")]
        csrc = os.path.join(_HERE, "..", "..", "vkfft_b200", "csrc")
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call([os.path.join(_HERE, "build_cluster.sh")])
        _LIB = ctypes.CDLL(so)
        _LIB.emu_cluster_exec_plan.restype = ctypes.c_int
        _LIB.emu_selftest_cluster_checkers.restype = ctypes.c_int
    return _LIB


def set_cluster_capable(on):
    """make the emulated planner see a device that can run thread-block clusters (off by default: today's plans)"""
    lib().emu_set_cluster_capable(int(bool(on)))


def describe(desc, inverse=-1):
    buf = ctypes.create_string_buffer(16384)
    rc = lib().emu_describe(ctypes.byref(desc), int(inverse), buf, len(buf))
    return rc, buf.value.decode()


def exec_plan(desc, inverse, buffer, inp=None, out=None):
    """the plan on host arrays; a Four-Step pair marked as one cluster launch runs through the cluster kernel"""
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    npass = ctypes.c_int(0)
    rc = lib().emu_cluster_exec_plan(ctypes.byref(desc), int(inverse), vp(buffer), vp(inp), vp(out), ctypes.byref(npass))
    return rc, npass.value


def selftest_checkers(mode):
    return lib().emu_selftest_cluster_checkers(int(mode))


make_desc = emu.make_desc
