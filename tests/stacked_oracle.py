"""CPU oracle of the policy with a stacked recurrent core (``num_layers`` > 1), for the num_layers tests.

``oracle.ref_policy.RefPolicy`` restates the reference network, whose recurrent core is one ``nn.GRU`` layer.  This
subclass creates the same modules in the same order, with torch's own multi-layer ``nn.GRU`` / ``nn.LSTM(num_layers=L)``
in place of the single layer, so the stacked recurrence the CUDA path is compared with is stock torch, not a
restatement of it.  ``forward`` / ``sequence`` are RefPolicy's: the multi-layer torch module takes and returns ``[L, B, H]``
states.  At L = 1 it is RefPolicy, parameter for parameter (``test_num_layers_host.py``).
"""
import torch
import torch.nn as nn

from oracle import ref_optimizer as RO
from oracle.ref_policy import UNIT_GROUPS, RefPolicy


class StackedRefPolicy(RefPolicy):
    def __init__(self, hidden_size=256, cell="gru", num_layers=1):
        nn.Module.__init__(self)
        assert cell in ("gru", "lstm") and num_layers >= 1
        self.hidden_size, self.cell, self.num_layers = hidden_size, cell, num_layers
        H = hidden_size
        # creation order of RefPolicy.__init__ (policy.py:54-75), so a seeded construction draws the same numbers
        self.affine_env = nn.Linear(3, 128)
        self.affine_unit_basic_stats = nn.Linear(12, 128)
        for suffix, _, _ in UNIT_GROUPS:
            setattr(self, "affine_unit_" + suffix, nn.Linear(128, 128))
        self.affine_pre_rnn = nn.Linear(896, H)
        rnn_cls = nn.GRU if cell == "gru" else nn.LSTM
        self.rnn = rnn_cls(input_size=H, hidden_size=H, num_layers=num_layers, batch_first=True)
        self.affine_head_enum = nn.Linear(H, 4)
        self.affine_move_x = nn.Linear(H, 9)
        self.affine_move_y = nn.Linear(H, 9)
        self.affine_unit_attention = nn.Linear(H, 128)
        self.affine_head_ability = nn.Linear(H, 3)
        self.affine_value = nn.Linear(H, 1)

    def init_hidden(self):
        h = torch.zeros([self.num_layers, 1, self.hidden_size], dtype=torch.float32)
        return (h, torch.zeros_like(h)) if self.cell == "lstm" else h


def make_stacked_ref_optimizer(hidden_size=256, cell="gru", seq_len=16, num_layers=1, seed=7, **kw):
    """``torch.manual_seed(7); Policy(num_layers=L)`` + the reference optimizer step on the CPU."""
    torch.manual_seed(seed)
    return RO.RefOptimizer(StackedRefPolicy(hidden_size, cell, num_layers), seq_len=seq_len, **kw)
