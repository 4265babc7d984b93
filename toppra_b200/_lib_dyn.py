"""ctypes binding of libtoppra_b200_dyn.so (include/toppra_b200_dyn.h): rigid-body inverse dynamics (RNEA) of a
fixed-base tree, the motor side of its geared drives, the wrench across a joint, the kinetic energy and momentum of
the whole tree, and linearly coupled joints (URDF mimic joints).

The companion library links against libtoppra_b200.so and reports errors through its tb_last_error(), so errors are
read with `_lib.check`.  There is NO CPU fallback: if the library is missing or a call fails, this module raises."""
import ctypes
import os

from . import _lib

LIB_PATH = os.path.join(_lib._HERE, "libtoppra_b200_dyn.so")

_c_dp = ctypes.c_void_p
_int = ctypes.c_int
_stream = ctypes.c_void_p

_PROTOS = {
    "tbd_version": ([], _int),
    "tbd_rnea": ([_c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_torque_terms": ([_c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_frame_velocity": ([_c_dp, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_velocity_norm_terms": ([_c_dp, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_frame_acceleration": ([_c_dp, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_acceleration_terms": ([_c_dp, _int, _c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_contact_wrench": ([_c_dp, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_contact_wrench_terms": ([_c_dp, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream],
                                 _int),
    "tbd_frame_inverse_inertia": ([_c_dp, _int, _c_dp, _int, _c_dp, _c_dp, _stream], _int),
    "tbd_collision_energy_terms": ([_c_dp, _int, _c_dp, ctypes.c_double, _int, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_support_wrench": ([_c_dp, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_support_wrench_terms": ([_c_dp, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream],
                                 _int),
    "tbd_separation": ([_c_dp, _int, _c_dp, _int, _int, _int, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream],
                       _int),
    "tbd_separation_terms": ([_c_dp, _int, _c_dp, _int, _int, _int, _int, ctypes.c_double, ctypes.c_double,
                              ctypes.c_double, ctypes.c_double, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_capsule_separation": ([_c_dp, _int, _c_dp, _int, _int, _int, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp,
                                _stream], _int),
    "tbd_capsule_separation_terms": ([_c_dp, _int, _c_dp, _int, _int, _int, _int, ctypes.c_double, ctypes.c_double,
                                      ctypes.c_double, ctypes.c_double, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream],
                                     _int),
    "tbd_drive_torque": ([_c_dp, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_drive_torque_terms": ([_c_dp, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_drive_speed_terms": ([_int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _stream], _int),
    "tbd_joint_wrench": ([_c_dp, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_joint_wrench_terms": ([_c_dp, _int, _c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream],
                               _int),
    "tbd_energy_momentum": ([_c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_energy_momentum_terms": ([_c_dp, _int, _int, _int, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_coupled_rnea": ([_c_dp, _int, _c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
    "tbd_coupled_torque_terms": ([_c_dp, _int, _c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp,
                                  _stream], _int),
    "tbd_coupling_expand": ([_int, _c_dp, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _stream], _int),
}

_dlib = None


def load():
    """Load libtoppra_b200_dyn.so (after libtoppra_b200.so, whose error slot it shares)."""
    global _dlib
    if _dlib is None:
        _lib.load()
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "toppra_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (argtypes, restype) in _PROTOS.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing: loud on purpose
            fn.argtypes = argtypes
            fn.restype = restype
        _dlib = lib
    return _dlib


def exported_symbols():
    return sorted(_PROTOS)
