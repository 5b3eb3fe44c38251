"""g2vec_b200 -- H100-native implementation of G2Vec's two data-parallel hot paths
(step 3 random-walk generator, step 4 modified-CBOW trainer; mathcom/G2Vec G2Vec.py:324-352, 217-286)
behind the reference's call sites and CLI.  Hand-written sm_90a CUDA reached through a C ABI
(include/g2vec_b200.h); torch is used for device memory, streams and torch.distributed only.
"""
from .walks import WalkGraph, generate_paths, generate_paths_host, generate_pathSet, walk_bias  # noqa: F401
from .cbow import train_cbow, compute_genetovec, cbow_step_host, CbowModel, WindowFeeder  # noqa: F401
from .perm import perm_test  # noqa: F401
from .neighbors import nearest_genes  # noqa: F401
from .kmeans import kmeans_lgroups  # noqa: F401
from .tsne import tsne_map  # noqa: F401
from .gsea import gsea, read_gmt  # noqa: F401
from .signature import signature_cv  # noqa: F401
from .diffcoex import diffcoex_test  # noqa: F401
from .netrank import netrank_test  # noqa: F401
from .lasso import lasso_cv  # noqa: F401
from .survival import survival_test, read_survival  # noqa: F401
from . import survival_cv  # noqa: F401  (the module: g2vec_b200.survival_cv.survival_cv runs the test)
from . import graph, paths  # noqa: F401

__version__ = "0.1.0"
