"""CPU: fcn_mega_forward rejects a layer table whose tile width or K atoms per stage the kernel was not built for
(the kernel derives the K atoms from the tile width at compile time).  Validation runs before any CUDA call."""
import ctypes as C

import pytest


def _args(NT, k_atoms):
    from frustum_convnet_b200 import _lib
    layer = _lib.MegaLayer(NT=NT, k_atoms=k_atoms, n_stage=1)
    dummy = (C.c_int * 16)()
    a = _lib.MegaArgs(n_layers=1, n_jobs=0, n_flags=0, layers=C.addressof(layer), jobs=C.addressof(dummy),
                      tmaps=C.addressof(dummy), sync=C.addressof(dummy), n_maps=1, NH=12, NS=8)
    return a, layer


@pytest.mark.parametrize("NT,k_atoms,ok", [(256, 1, True), (128, 2, True), (64, 2, True),
                                           (256, 2, False), (128, 1, False), (64, 1, False), (96, 2, False)])
def test_mega_layer_table_validation(NT, k_atoms, ok):
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    a, _layer = _args(NT, k_atoms)
    rc = lib.fcn_mega_forward(C.byref(a), None)
    if ok:
        assert rc == 0                       # n_jobs = 0: nothing is launched
    else:
        assert rc == -1 and b"k_atoms" in lib.fcn_last_error()
