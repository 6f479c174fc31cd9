"""Batched gradients without a GPU: network_function refuses a bad `batched` argument before it compiles anything, and
the new entry points are declared with the signatures the header gives them."""
import ctypes as C

import numpy as np
import pytest


def small_net():
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    a = Tensor([0, 1], [2, 2])
    a.set_tensor_data(TensorData.Matrix(np.eye(2)))
    b = Tensor([1, 2], [2, 2])
    b.set_tensor_data(TensorData.Gate("h"))
    c = Tensor([2, 0], [2, 2])
    c.set_tensor_data(TensorData.Matrix(np.eye(2)))
    return Tensor.new_composite([a, b, c]), ContractionPath.simple([(0, 1), (0, 2)])


@pytest.mark.parametrize("kwargs,match", [
    (dict(wrt=[0], batched=[0], sliced_legs=[1]), "sliced_legs"),
    (dict(wrt=[0], batched=[1]), "Matrix"),                     # a gate leaf cannot take per-instance payloads
    (dict(wrt=[0], batched=[2, 2]), "twice"),
    (dict(wrt=[0], batched=[3]), "Matrix"),                     # no such leaf
])
def test_network_function_refuses_bad_batched(kwargs, match):
    pytest.importorskip("torch")
    from tnc_b200.autograd import network_function
    tn, path = small_net()
    with pytest.raises(ValueError, match=match):
        network_function(tn, path, **kwargs)


def test_batched_signatures():
    from tnc_b200._lib import SIGNATURES
    vpp = C.POINTER(C.c_void_p)
    assert SIGNATURES["tncb_plan_vjp_batch"] == (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, vpp, vpp, vpp])
    assert SIGNATURES["tncb_plan_stage_batch"][1][:3] == [C.c_void_p, C.c_void_p, C.c_size_t]
