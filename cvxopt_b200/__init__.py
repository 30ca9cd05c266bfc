"""cvxopt_b200 — H100-native KKT hot path for CVXOPT's cone solvers.

Only what the path needs: the C-ABI CUDA library (csrc/, libcvxopt_b200.so) and
the host-side mirror of the reference's kktsolver / misc_solvers interface.
"""
from ._lib import load, exported_symbols, LIB_PATH  # noqa: F401
from .kkt import kkt_chol, kkt_chol2, kkt_ldl2, kkt_qr, KKTChol, cp_kktsolver, cpl_kktsolver  # noqa: F401
from . import scaling  # noqa: F401
from .conelp import conelp  # noqa: F401
from .batch import QPBatch, QPBatchGroup, qp_batch, qp_batch_distributed, shard_bounds, shard_indices  # noqa: F401
from .batch import ConeLPBatch, ConeLPBatchGroup, conelp_batch  # noqa: F401
from .batch import SDPBatch, SDPBatchGroup, sdp_batch  # noqa: F401
from .batch import SDPQPBatch, SDPQPBatchGroup, coneqp_batch  # noqa: F401
from .batch import GPBatch, GPBatchGroup, gp_batch  # noqa: F401
from .batch import CPBatch, CPBatchGroup, cp_batch  # noqa: F401
from .batch import CPLBatch, CPLBatchGroup, cpl_batch  # noqa: F401
from .batch import SDPCPLBatch, SDPCPLBatchGroup, sdp_cpl_batch  # noqa: F401
from .batch import QCQPBatch, QCQPBatchGroup, qcqp_batch  # noqa: F401

__all__ = ["kkt_chol", "kkt_chol2", "kkt_ldl2", "kkt_qr", "KKTChol", "cp_kktsolver", "cpl_kktsolver", "QPBatch", "qp_batch", "conelp", "qp_batch_distributed", "load",
           "ConeLPBatch", "conelp_batch", "SDPBatch", "SDPBatchGroup", "sdp_batch",
           "SDPQPBatch", "SDPQPBatchGroup", "coneqp_batch", "GPBatch", "GPBatchGroup", "gp_batch",
           "CPBatch", "CPBatchGroup", "cp_batch",
           "CPLBatch", "CPLBatchGroup", "cpl_batch",
           "SDPCPLBatch", "SDPCPLBatchGroup", "sdp_cpl_batch",
           "QCQPBatch", "QCQPBatchGroup", "qcqp_batch", "qp_layer", "qcqp_layer",
           "coneqp_layer", "conelp_layer", "gp_layer", "cp_layer", "cpl_layer",
           "device_count", "launch_count"]


def __getattr__(name):
    # the layers import torch, which `import cvxopt_b200` does not need otherwise
    if name in ("qp_layer", "qcqp_layer", "coneqp_layer", "conelp_layer", "gp_layer", "cp_layer", "cpl_layer"):
        from . import layer
        return getattr(layer, name)
    raise AttributeError("module 'cvxopt_b200' has no attribute %r" % name)


def device_count():
    return load().cvxb_device_count()


def launch_count():
    return int(load().cvxb_launch_count())
