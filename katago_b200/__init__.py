"""katago_b200 - H100-native (sm_90a) implementation of KataGo's self-play hot path behind KataGo's own interfaces.

Only what the path needs lives here: csrc/ (CUDA kernels + the C ABI in include/kgb200.h), nn_backend.py (host-side
mirror of the reference's `namespace NeuralNet`, cpp/neuralnet/nninterface.h), modelgen.py (synthetic model files).
"""
from .nn_backend import (  # noqa: F401
    ComputeContext, ComputeHandle, KGBError, LoadedModel, NeuralNet, SelfPlay, board_replay, library_path, load_library, zobrist_tables,
)
