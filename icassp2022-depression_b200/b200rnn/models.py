"""Host-side mirror of the reference's model classes for the hot path, built on the b200rnn GRU / LSTM.

Same class names, constructor arguments, attribute / state-dict key names and ``forward`` semantics as

* ``AudioBiLSTM``  Classification/audio_gru_whole.py:24-108, Regression/audio_bilstm_perm.py:45-127
* ``TextBiLSTM``   Classification/text_bilstm_whole.py:23-114, Regression/text_bilstm_perm.py:37-124
* ``fusion_net``   Classification/fuse_net_whole.py:245-374,   Regression/fuse_net.py:224-351
* ``MyLoss``       Classification/fuse_net_whole.py:376-395,   Regression/fuse_net.py:353-366

so the reference training loops (``train()`` audio_gru_whole.py:161-201, text_bilstm_whole.py:154-193,
fuse_net_whole.py:421-465) run on them unchanged. Only the sequence encoders differ: ``self.lstm_net_audio``
is a :class:`b200rnn.GRU`, ``self.lstm_net`` a :class:`b200rnn.LSTM`. The dense shells around them stay
ordinary PyTorch modules (SURVEY.md §8f ranks their fusion as "next").

The two flavours of each class (classification / regression script) are selected with ``regression=``.
"""
from __future__ import annotations

from typing import Sequence, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from .modules import GRU, LSTM
from .staging import FuseBatch, stage_fuse_batch


def attention_pool(attention_layer: nn.Module, seq_out: torch.Tensor, last_hidden: torch.Tensor) -> torch.Tensor:
    """``attention_net_with_w`` (text_bilstm_whole.py:74-99).

    seq_out [B,T,2H] (fwd | rev halves), last_hidden [B, L*D, H]  ->  context [B,H]
    """
    fwd, rev = torch.chunk(seq_out, 2, dim=-1)
    h = fwd + rev                                            # [B,T,H]
    query = attention_layer(last_hidden.sum(dim=1, keepdim=True))  # [B,1,H]
    scores = torch.bmm(query, torch.tanh(h).transpose(1, 2))       # [B,1,T]
    return torch.bmm(F.softmax(scores, dim=-1), h).squeeze(1)


def _attention_layer(hidden: int) -> nn.Sequential:
    return nn.Sequential(nn.Linear(hidden, hidden), nn.ReLU(inplace=True))


def _init_xavier(module: nn.Module, skip_ln: bool) -> None:
    """``init_weight`` of the text models (text_bilstm_whole.py:37-43 / text_bilstm_perm.py:51-56)."""
    for name, param in module.named_parameters():
        if skip_ln and "ln" in name:
            continue
        if "bias" in name:
            nn.init.constant_(param, 0.0)
        elif "weight" in name:
            nn.init.xavier_uniform_(param)


class AudioBiLSTM(nn.Module):
    """Audio branch: [LayerNorm ->] 2-layer GRU -> mean/sum over time -> MLP head."""

    def __init__(self, config: dict, regression: bool = False):
        super().__init__()
        self.regression = regression
        self.num_classes = config["num_classes"]
        self.learning_rate = config.get("learning_rate")
        self.dropout = config["dropout"]
        self.hidden_dims = config["hidden_dims"]
        self.rnn_layers = config["rnn_layers"]
        self.embedding_size = config["embedding_size"]
        self.bidirectional = config.get("bidirectional", False)
        self.build_model()

    def build_model(self) -> None:
        H, p = self.hidden_dims, self.dropout
        self.attention_layer = _attention_layer(H)  # present (and saved) in the reference, unused in forward
        if self.regression:
            self.lstm_net_audio = GRU(self.embedding_size, H, num_layers=self.rnn_layers, dropout=p,
                                      bidirectional=self.bidirectional, batch_first=True)
            self.bn = nn.BatchNorm1d(3)             # audio_bilstm_perm.py:81 (unused in forward)
            tail: list = [nn.ReLU()]
        else:
            self.lstm_net_audio = GRU(self.embedding_size, H, num_layers=self.rnn_layers, dropout=p,
                                      batch_first=True)
            self.ln = nn.LayerNorm(self.embedding_size)
            tail = [nn.Softmax(dim=1)]
        self.fc_audio = nn.Sequential(nn.Dropout(p), nn.Linear(H, H), nn.ReLU(), nn.Dropout(p),
                                      nn.Linear(H, self.num_classes), *tail)

    def pooled(self, x: torch.Tensor) -> torch.Tensor:
        """[LayerNorm ->] GRU -> mean / sum over time, [B, H]."""
        if self.regression:                          # audio_bilstm_perm.py:122-125: GRU -> sum(dim=1)
            return self.lstm_net_audio.forward_ln_sum(x, None)
        # audio_gru_whole.py:103-106: LayerNorm -> GRU -> mean(dim=1); the shell is fused around the encoder
        return self.lstm_net_audio.forward_ln_sum(x, self.ln) * (1.0 / x.shape[1])

    def forward_logits(self, x: torch.Tensor) -> torch.Tensor:
        """``forward`` without the final activation (the input of the model's Softmax / ReLU): what a fused
        softmax + cross-entropy loss consumes (b200rnn.train_step)."""
        return self.fc_audio[:-1](self.pooled(x))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.fc_audio(self.pooled(x))


class TextBiLSTM(nn.Module):
    """Text branch: 2-layer BiLSTM -> attention pooling -> MLP head."""

    def __init__(self, config: dict, regression: bool = False):
        super().__init__()
        self.regression = regression
        self.num_classes = config["num_classes"]
        self.learning_rate = config.get("learning_rate")
        self.dropout = config["dropout"]
        self.hidden_dims = config["hidden_dims"]
        self.rnn_layers = config["rnn_layers"]
        self.embedding_size = config["embedding_size"]
        self.bidirectional = config.get("bidirectional", True)
        self.build_model()
        self.init_weight()

    def init_weight(self) -> None:
        _init_xavier(self, skip_ln=not self.regression)

    def build_model(self) -> None:
        H, p = self.hidden_dims, self.dropout
        self.attention_layer = _attention_layer(H)
        self.lstm_net = LSTM(self.embedding_size, H, num_layers=self.rnn_layers, dropout=p,
                             bidirectional=self.bidirectional)
        if self.regression:                          # text_bilstm_perm.py:75-83
            self.fc_out = nn.Sequential(nn.Dropout(p), nn.Linear(H, H), nn.ReLU(), nn.Dropout(p),
                                        nn.Linear(H, self.num_classes), nn.ReLU())
        else:                                        # text_bilstm_whole.py:60-71
            self.fc_out = nn.Sequential(nn.Linear(H, H), nn.ReLU(), nn.Dropout(p),
                                        nn.Linear(H, self.num_classes), nn.Softmax(dim=1))
            self.ln1 = nn.LayerNorm(self.embedding_size)
            self.ln2 = nn.LayerNorm(H)

    def attention_net_with_w(self, lstm_out: torch.Tensor, lstm_hidden: torch.Tensor) -> torch.Tensor:
        return attention_pool(self.attention_layer, lstm_out, lstm_hidden)

    def context(self, x: torch.Tensor) -> torch.Tensor:
        # [B,T,E] -> time-major NON-contiguous view, consumed in place by the kernels (text_bilstm_whole.py:103)
        seq, (h_n, _) = self.lstm_net(x.permute(1, 0, 2))
        from .fused_head import attention_pool_tm   # one kernel forward, one backward (SURVEY.md 8f rank 1)

        return attention_pool_tm(self.attention_layer, seq, h_n)

    def forward_logits(self, x: torch.Tensor) -> torch.Tensor:
        """``forward`` without the final activation (see AudioBiLSTM.forward_logits)."""
        return self.fc_out[:-1](self.context(x))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.fc_out(self.context(x))


class fusion_net(nn.Module):  # noqa: N801  (reference class name)
    """Late fusion of the two pretrained branches (fuse_net_whole.py:245-374 / fuse_net.py:224-351)."""

    def __init__(self, text_embed_size, text_hidden_dims, rnn_layers, dropout, num_classes, audio_hidden_dims,
                 audio_embed_size, regression: bool = False):
        super().__init__()
        self.regression = regression
        self.text_embed_size = text_embed_size
        self.audio_embed_size = audio_embed_size
        self.text_hidden_dims = text_hidden_dims
        self.audio_hidden_dims = audio_hidden_dims
        self.rnn_layers = rnn_layers
        self.dropout = dropout
        self.num_classes = num_classes
        Ht, Ha, p = text_hidden_dims, audio_hidden_dims, dropout

        self.attention_layer = _attention_layer(Ht)
        self.lstm_net = LSTM(text_embed_size, Ht, num_layers=rnn_layers, dropout=p, bidirectional=True)
        self.fc_out = nn.Sequential(nn.Dropout(p), nn.Linear(Ht, Ht), nn.ReLU(), nn.Dropout(p))

        self.lstm_net_audio = GRU(audio_embed_size, Ha, num_layers=rnn_layers, dropout=p, bidirectional=False,
                                  batch_first=True)
        self.fc_audio = nn.Sequential(nn.Dropout(p), nn.Linear(Ha, Ha), nn.ReLU(), nn.Dropout(p))
        if not regression:
            self.ln = nn.LayerNorm(audio_embed_size)  # fuse_net_whole.py:295

        self.modal_attn = nn.Linear(Ht + Ha, Ht + Ha, bias=False)
        self.fc_final = nn.Sequential(nn.Linear(Ht + Ha, num_classes, bias=False),
                                      nn.ReLU() if regression else nn.Softmax(dim=1))

    def attention_net_with_w(self, lstm_out: torch.Tensor, lstm_hidden: torch.Tensor) -> torch.Tensor:
        return attention_pool(self.attention_layer, lstm_out, lstm_hidden)

    def pretrained_feature(self, x: Union[FuseBatch, Sequence]):
        """(text_feature [B,Ht], audio_feature [B,Ha]) under ``no_grad`` (fuse_net_whole.py:336-366).

        ``x`` is the reference's python list of ``[audio(T,Ea), text(T,Et)]`` pairs, or a pre-staged
        :class:`b200rnn.staging.FuseBatch` of device tensors (the list is staged through pinned memory in one
        copy per modality instead of ``torch.tensor(list)``, fuse_net_whole.py:343).
        """
        with torch.no_grad():
            batch = x if isinstance(x, FuseBatch) else stage_fuse_batch(x, self.fc_final[0].weight.device)
            from .fused_head import attention_pool_tm

            seq, (h_n, _) = self.lstm_net(batch.text.permute(1, 0, 2))
            text_feature = self.fc_out(attention_pool_tm(self.attention_layer, seq, h_n))

            # LayerNorm (classification flavour only) -> GRU -> sum over time, fused around the encoder
            pooled = self.lstm_net_audio.forward_ln_sum(batch.audio, None if self.regression else self.ln)
            audio_feature = self.fc_audio(pooled)
        return text_feature, audio_feature

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.regression:                          # fuse_net.py:345-351
            x = torch.sigmoid(self.modal_attn(x)) * x
        return self.fc_final(x)


class MyLoss(nn.Module):
    """Two-head loss on the halves of ``fc_final[0].weight`` (fuse_net_whole.py:380-395 / fuse_net.py:357-366).

    The reference reads ``config['text_hidden_dims']`` from a module global; here it is a constructor argument.
    """

    def __init__(self, text_hidden_dims: int = 128, regression: bool = False):
        super().__init__()
        self.text_hidden_dims = text_hidden_dims
        self.regression = regression

    def forward(self, text_feature, audio_feature, target, model):
        weight = model.fc_final[0].weight
        k = self.text_hidden_dims
        pred_text = F.linear(text_feature, weight[:, :k])
        pred_audio = F.linear(audio_feature, weight[:, k:])
        target = torch.as_tensor(target, device=pred_text.device)
        if self.regression:
            target = target.view_as(pred_text).float()
            return F.smooth_l1_loss(pred_text, target) + F.smooth_l1_loss(pred_audio, target)
        return F.cross_entropy(pred_text, target) + F.cross_entropy(pred_audio, target)
