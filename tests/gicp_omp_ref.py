"""Shared by the pclomp GICP tests: the sequential CPU reference of pclomp::GeneralizedIterativeClosestPoint (tests/gicp_omp_ref.cpp,
compiled into a temporary directory).  It is gicp_pcl_ref.Reference with pclomp's functor pose: cost, fdf and align run the
ref_gicp_omp_* entry points; covariances, correspondences and apply_state are GICP's."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

import gicp_pcl_ref as gr

SRC = os.path.join(gr.ROOT, "tests", "gicp_omp_ref.cpp")
_VP = C.c_void_p
_SZ = C.c_size_t
_OMP = {"ref_gicp_pcl_cost": "ref_gicp_omp_cost", "ref_gicp_pcl_fdf": "ref_gicp_omp_fdf", "ref_gicp_pcl_align": "ref_gicp_omp_align"}


class _Lib:
    """the library under the names gicp_pcl_ref.Reference calls, its pose-dependent ones bound to pclomp's entry points"""

    def __init__(self, L):
        self._L = L

    def __getattr__(self, name):
        return getattr(self._L, _OMP.get(name, name))


class Reference(gr.Reference):
    def __init__(self, tmpdir):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        so = os.path.join(str(tmpdir), "libgicp_omp_ref.so")
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-variable", "-o", so, SRC])
        L = C.CDLL(so)
        L.ref_gicp_pcl_covariances.argtypes = [_VP, _SZ, _SZ, C.c_int, _VP]
        pair = [_VP, _SZ, _SZ, _VP, _VP, _SZ, _SZ, _VP, _VP]
        L.ref_gicp_pcl_correspondences.restype = _SZ
        L.ref_gicp_pcl_correspondences.argtypes = pair + [_VP, C.c_double, _VP, _VP]
        for pre in ("ref_gicp_pcl", "ref_gicp_omp"):  # the library carries pcl GICP's entry points too
            getattr(L, pre + "_cost").restype = _SZ
            getattr(L, pre + "_cost").argtypes = pair + [_VP, C.c_double, _VP, _VP]
            getattr(L, pre + "_fdf").restype = _SZ
            getattr(L, pre + "_fdf").argtypes = pair + [_VP, C.c_double, _VP, _VP, _VP]
            getattr(L, pre + "_align").restype = _SZ
            getattr(L, pre + "_align").argtypes = pair + [_VP, _VP, _VP, _VP, _VP, _SZ]
        L.ref_gicp_pcl_apply_state.argtypes = [_VP, _VP]
        L.ref_gicp_omp_pose.argtypes = [_VP, _VP, _VP]
        self.lib = _Lib(L)

    def pose(self, x, guess):
        """applyState(guess, x): the pose pclomp's functor evaluates at x (row-major float32 4x4)"""
        xv = np.ascontiguousarray(x, np.float64)
        g = gr._row(guess)
        T = np.empty((4, 4), np.float32)
        self.lib.ref_gicp_omp_pose(gr._p(xv), gr._p(g), gr._p(T))
        return T
