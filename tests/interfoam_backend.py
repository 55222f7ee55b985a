"""Dry-run aid for rapidcfd-dev_b200/interfoam.py (NOT part of the product): the oracle-backed stand-in of tests/oracle_backend.py
with the two entry points of csrc/vof.cu answered by oracle/interfoam_oracle.py, so that the sequencing of the phase-fraction step
runs on the CPU.  It says nothing about the CUDA path."""
import numpy as np

from oracle import interfoam_oracle as io
from oracle_backend import FieldOps, _Capi, _Ctx, _np


class Capi(_Capi):
    @staticmethod
    def fv_limited_flux(addr, scheme, faceFlux, vf, gradc, centres, cdWeights, k=1.0, fluxSign=1, outSign=1):
        g = None if gradc is None else _np(gradc).reshape(-1, 3)
        return FieldOps._t(io.limited_flux(scheme, addr.o.lower(), addr.o.upper(), _np(faceFlux), _np(vf), g, _np(centres).reshape(-1, 3),
                                           _np(cdWeights), k, fluxSign, outSign))

    @staticmethod
    def vof_interface_flux(addr, w, gradAlpha, Sf, bSf, bSnGrad, deltaN, phi=None, magSf=None, cAlpha=0.0):
        nHatf, nHatfB, phir = io.interface_flux(addr.o.lower(), addr.o.upper(), _np(w), _np(gradAlpha), _np(Sf), addr.bfc, _np(bSf),
                                                _np(bSnGrad), deltaN, _np(phi), _np(magSf), cAlpha)
        return FieldOps._t(nHatf), FieldOps._t(nHatfB), None if phir is None else FieldOps._t(phir)


def fixture():
    """(capi, ctx, torch) as the `gpu` fixtures yield them"""
    import torch
    return Capi, _Ctx(), torch
