"""code2vec_b200: H100-native (sm_90a) backend for code2vec's path-attention hot path.

Layout: ``csrc/`` CUDA kernels + the C ABI (include/c2v_b200.h) -> ``libc2v_b200.so``;
``engine.py`` ctypes binding + storage; the host-side mirror of the reference's model / config /
reader interface lives beside it (``config.py``, ``vocabularies.py``, ``path_context_reader.py``,
``model_base.py``, ``b200_model.py``).
"""
__version__ = "0.1.0"


def load_model_dynamically(config):
    """The reference's backend factory (code2vec.py:7-13) for the two backends built here."""
    if config.DL_FRAMEWORK == "b200":
        from .b200_model import Code2VecModel
    elif config.DL_FRAMEWORK == "b200-keras":
        from .b200_keras_model import Code2VecModel
    else:
        raise ValueError("framework %r is the reference's own backend; this package provides 'b200' and 'b200-keras'"
                         % (config.DL_FRAMEWORK,))
    return Code2VecModel(config)
