"""b200rnn — H100-native (sm_90a) GRU / BiLSTM sequence encoders behind the torch.nn.GRU / nn.LSTM API (and
nn.RNN, the cells GRUCell / LSTMCell / RNNCell).

The one hot path of speechandlanguageprocessing/ICASSP2022-Depression (SURVEY.md §8), rebuilt from scratch:
PyTorch host code -> C-ABI shared library (include/b200rnn.h) -> hand-written CUDA kernels.
Importing this package does not need a GPU; running any op does, and fails loudly without one.
"""
from . import _lib
from . import ops  # registers the b200rnn:: custom ops (torch.export / torch.compile)
from ._lib import B200RNNError
from .modules import GRU, LSTM, RNN, GRUCell, LSTMCell, RNNCell, from_torch, install, uninstall
from .functional import RNNConfig, gemm, rnn_forward
from .staging import FuseBatch, PinnedStager, bind_host_thread_to_gpu_numa_node, stage_fuse_batch
from .dp import GradBucket, broadcast_parameters, shard_batch
from .models import AudioBiLSTM, MyLoss, TextBiLSTM, attention_pool, fusion_net
from .fused_head import FusedFuseStep
from .optim import FlatAdamW
from .train_step import FuseFineTuneStep, TrainStep, softmax_cross_entropy
from .dp import PeerComm

__all__ = [
    "GRU", "LSTM", "RNN", "GRUCell", "LSTMCell", "RNNCell", "install", "uninstall", "from_torch", "rnn_forward", "gemm", "RNNConfig", "B200RNNError",
    "AudioBiLSTM", "TextBiLSTM", "fusion_net", "MyLoss", "attention_pool", "FuseBatch", "PinnedStager",
    "stage_fuse_batch", "GradBucket", "broadcast_parameters", "shard_batch", "FusedFuseStep", "FlatAdamW",
    "TrainStep", "FuseFineTuneStep", "softmax_cross_entropy", "PeerComm",
]
