from .tensor import Tensor
from .tensordata import TensorData
from .contraction import contract_tensor_network, leaves, NetworkPlan, PreparedNetwork

__all__ = ["Tensor", "TensorData", "contract_tensor_network", "leaves", "NetworkPlan", "PreparedNetwork"]
