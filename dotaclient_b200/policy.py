"""``Policy`` -- drop-in for the reference's ``policy.py`` on the optimizer hot path.

Same constructor-created parameters, same ``state_dict`` (34 keys, shapes and order of
``policy.py:54-75``), same ``forward`` signature and outputs (``policy.py:92-167``); the recurrent
layer runs through the hand-written sm_90a recurrence kernels (``dotaclient_b200/csrc``), and the
unit encoder through the fused encoder kernel when it is available.  Three additions, all
keyword-only so ``Policy()`` is the reference's network: ``hidden_size`` (reference: 256),
``cell`` ('gru' = the reference's ``nn.GRU``, 'lstm' = the cell BASELINE.json names) and
``num_layers`` (reference: 1), the depth of the recurrent core with the semantics of
``nn.GRU(num_layers=L)``: layer k consumes layer k-1's output sequence, every hidden state is
``[L, B, H]`` and the ``state_dict`` carries ``rnn.*_l{k}`` for every layer (34 + 4(L-1) keys).

Every ``hidden_size`` that is a multiple of 32 runs on the GPU: 128, 256 and the other multiples of 128 on their
dedicated recurrence kernels, the rest (64, 96, 160, 192, ...) on the generic ones.  Any width constructs, so that a
``state_dict`` of any width can be held or converted on the CPU; the first CUDA forward of another width raises the
GEMM's ``DC_EUNSUPPORTED`` error.

CUDA only: calling ``forward`` with CPU tensors raises (there is no CPU fallback).
"""
import logging
import re

import numpy as np
import torch
import torch.nn as nn

from . import encoder_ops, ops

logger = logging.getLogger(__name__)

eps = np.finfo(np.float32).eps.item()          # policy.py:15
TICKS_PER_OBSERVATION = 15                      # policy.py:17
REWARD_KEYS = ['enemy', 'win', 'xp', 'hp', 'kills', 'death', 'lh', 'denies', 'tower_hp', 'mana']  # policy.py:20
MAX_VALUE_HEADS = len(REWARD_KEYS)             # one value head per reward group (DotaOptimizer(value_heads=...))

# (parameter suffix, observation key, units per step) in concatenation order (policy.py:99-131)
UNIT_GROUPS = (("ah", "allied_heroes", 1), ("eh", "enemy_heroes", 5), ("anh", "allied_nonheroes", 16),
               ("enh", "enemy_nonheroes", 16), ("ath", "allied_towers", 1), ("eth", "enemy_towers", 1))


class MaskedCategorical:
    """Masked categorical over log-probs (``policy.py:23-33``)."""

    def __init__(self, log_probs, mask):
        self.log_probs = log_probs
        self.mask = mask.bool()
        self.masked_probs = torch.exp(log_probs).masked_fill(~self.mask, 0.)

    def sample(self):
        return torch.multinomial(self.masked_probs[-1], num_samples=1)


class _RnnParams(nn.Module):
    """Parameter holder with ``nn.GRU``/``nn.LSTM`` names and order (``weight_ih_l{k}, weight_hh_l{k}, bias_ih_l{k},
    bias_hh_l{k}`` for every layer k) so ``rnn.weight_ih_l0`` ... load unchanged."""

    def __init__(self, template):
        super().__init__()
        self.num_layers = template.num_layers
        for k in range(self.num_layers):
            for name in ("weight_ih_l%d" % k, "weight_hh_l%d" % k, "bias_ih_l%d" % k, "bias_hh_l%d" % k):
                self.register_parameter(name, nn.Parameter(getattr(template, name).detach().clone()))

    def layer(self, k):
        """(w_ih, w_hh, b_ih, b_hh) of layer ``k``."""
        return tuple(getattr(self, "%s_l%d" % (n, k)) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))


class Policy(nn.Module):
    TICKS_PER_SECOND = 30
    MAX_MOVE_SPEED = 550
    MAX_MOVE_IN_OBS = (MAX_MOVE_SPEED / TICKS_PER_SECOND) * TICKS_PER_OBSERVATION
    N_MOVE_ENUMS = 9
    MOVE_ENUMS = (np.arange(N_MOVE_ENUMS, dtype=np.float32) - int(N_MOVE_ENUMS / 2)) \
        * (MAX_MOVE_IN_OBS / (N_MOVE_ENUMS - 1) * 2)                                    # policy.py:42-43
    OBSERVATIONS_PER_SECOND = TICKS_PER_SECOND / TICKS_PER_OBSERVATION
    MAX_UNITS = 1 + 5 + 16 + 16 + 1 + 1
    ACTION_OUTPUT_COUNTS = {'enum': 4, 'x': 9, 'y': 9, 'target_unit': MAX_UNITS, 'ability': 3}
    OUTPUT_KEYS = ACTION_OUTPUT_COUNTS.keys()
    INPUT_KEYS = ['env', 'allied_heroes', 'enemy_heroes', 'allied_nonheroes', 'enemy_nonheroes',
                  'allied_towers', 'enemy_towers']

    def __init__(self, *, hidden_size=256, cell="gru", num_layers=1, value_heads=1):
        super().__init__()
        if cell not in ("gru", "lstm"):
            raise ValueError("cell must be 'gru' or 'lstm'")
        if int(num_layers) != num_layers or num_layers < 1:
            raise ValueError("num_layers must be an integer >= 1, got %r" % (num_layers,))
        if isinstance(value_heads, bool) or int(value_heads) != value_heads or not 1 <= value_heads <= MAX_VALUE_HEADS:
            raise ValueError("value_heads must be an integer in [1, %d], got %r" % (MAX_VALUE_HEADS, value_heads))
        self.value_heads = int(value_heads)
        self.hidden_size = H = int(hidden_size)
        self.cell = cell
        self.num_layers = int(num_layers)
        # Creation order == reference (policy.py:54-75) so torch.manual_seed(7); Policy() reproduces its init.
        self.affine_env = nn.Linear(3, 128)
        self.affine_unit_basic_stats = nn.Linear(12, 128)
        for suffix, _, _ in UNIT_GROUPS:
            setattr(self, "affine_unit_" + suffix, nn.Linear(128, 128))
        self.affine_pre_rnn = nn.Linear(896, H)
        template = (nn.GRU if cell == "gru" else nn.LSTM)(input_size=H, hidden_size=H, num_layers=self.num_layers,
                                                          batch_first=True)
        self.rnn = _RnnParams(template)
        self.affine_head_enum = nn.Linear(H, 4)
        self.affine_move_x = nn.Linear(H, self.N_MOVE_ENUMS)
        self.affine_move_y = nn.Linear(H, self.N_MOVE_ENUMS)
        self.affine_unit_attention = nn.Linear(H, 128)
        self.affine_head_ability = nn.Linear(H, 3)
        self.affine_value = nn.Linear(H, self.value_heads)      # created last: value_heads leaves every other init as is

    @classmethod
    def from_state_dict(cls, state_dict):
        """The ``Policy`` a ``state_dict`` describes, loaded strictly: ``hidden_size`` from the rows of
        ``affine_pre_rnn.weight``, ``num_layers`` from the ``rnn.weight_hh_l{k}`` keys, ``cell`` from the rows of
        ``rnn.weight_hh_l0`` (3H: 'gru', 4H: 'lstm') and ``value_heads`` from the rows of ``affine_value.weight``.  Raises
        ``ValueError`` for a dict that is not a ``Policy``'s (missing keys, unexpected keys or shapes)."""
        try:
            H = int(state_dict['affine_pre_rnn.weight'].shape[0])
            rows = int(state_dict['rnn.weight_hh_l0'].shape[0])
            value_heads = int(state_dict['affine_value.weight'].shape[0])
        except (KeyError, TypeError, AttributeError, IndexError) as e:
            raise ValueError("not a Policy state_dict: %r" % (e,)) from None
        num_layers = sum(1 for k in state_dict if re.fullmatch(r'rnn\.weight_hh_l\d+', k))
        cells = {3 * H: 'gru', 4 * H: 'lstm'}
        if rows not in cells:
            raise ValueError("not a Policy state_dict: rnn.weight_hh_l0 has %d rows, neither 3 nor 4 x hidden_size %d"
                             % (rows, H))
        if not 1 <= value_heads <= MAX_VALUE_HEADS:
            raise ValueError("not a Policy state_dict: affine_value.weight has %d rows" % value_heads)
        pol = cls(hidden_size=H, cell=cells[rows], num_layers=num_layers, value_heads=value_heads)
        try:
            pol.load_state_dict(state_dict, strict=True)
        except RuntimeError as e:
            raise ValueError("not a Policy state_dict: %s" % e) from None
        return pol

    # ------------------------------------------------------------------ reference API
    def init_hidden(self):
        """Zero state ``[L, 1, H]`` (``policy.py:77-78``, L = ``num_layers``); an ``(h, c)`` tuple for the LSTM."""
        h = torch.zeros([self.num_layers, 1, self.hidden_size], dtype=torch.float32)
        return (h, torch.zeros_like(h)) if self.cell == "lstm" else h

    def single(self, hidden, **kwargs):
        """One step of one sequence (``policy.py:80-84``)."""
        for k in kwargs:
            kwargs[k] = kwargs[k].unsqueeze(0).unsqueeze(0)
        return self.__call__(**kwargs, hidden=hidden)

    def sequence(self, hidden, **kwargs):
        """One whole sequence (``policy.py:86-90``)."""
        for k in kwargs:
            kwargs[k] = kwargs[k].unsqueeze(0)
        return self.__call__(**kwargs, hidden=hidden)

    def forward(self, env, allied_heroes, enemy_heroes, allied_nonheroes, enemy_nonheroes,
                allied_towers, enemy_towers, hidden):
        """Batch-first ``(b, s, ...)`` inputs -> (logits dict ``(b, s, n)``, value ``(b, s, K)`` with K = ``value_heads``,
        hidden).  ``hidden`` is
        ``[L, b, H]`` (an ``(h, c)`` pair for the LSTM) in and out: as in torch, not batch-first."""
        return self._run((env, allied_heroes, enemy_heroes, allied_nonheroes, enemy_nonheroes,
                          allied_towers, enemy_towers), hidden, time_major=False)

    def forward_time_major(self, observations, hidden):
        """Same network on time-major ``(s, b, ...)`` inputs: the layout the recurrence kernels consume,
        so ``DotaOptimizer.train`` pays no transposes.  ``observations`` is a dict keyed by INPUT_KEYS."""
        return self._run(tuple(observations[k] for k in self.INPUT_KEYS), hidden, time_major=True)

    def _train_forward(self, observations, hidden, wait=None, reset=None, active=None):
        """The training step's forward on time-major inputs -> (the packed ``[S, B, ops.PACK_WIDTH]`` output of the four
        small heads and the value head, target-unit logits ``[S, B, 40]``): the tensors the fused PPO loss reads and
        backward starts from.  ``wait`` (see ``encoder_ops.unit_encoder``) lets the observations arrive while it runs.
        ``reset``: recurrent-state resets inside the sequences (``_recur``).  ``active``: see ``_head_outputs``; ``wait``
        is also called for its two tensors, right before the head."""
        x, unit_embedding = self._encode(observations['env'], [observations[k] for k in self.INPUT_KEYS[1:]], wait=wait)
        y, _ = self._recur(x.contiguous(), hidden, reset)
        if active is not None and wait is not None:
            for t in active:
                wait(t)
        return self._head_outputs(y, unit_embedding, active)

    # ------------------------------------------------------------------ implementation
    def _encode(self, env, groups, wait=None):
        """Observation encoders (``policy.py:97-138``) -> (x ``[..., H]``, encoder handle for the target-unit head): the explicit
        kernel chain of ``csrc/encoder.cu`` + wgmma GEMMs (no ``torch.cat``, no materialised ``[..., 40, 128]`` unit embedding)."""
        layers = [getattr(self, "affine_unit_" + s) for s, _, _ in UNIT_GROUPS]
        unit_embedding, x = encoder_ops.unit_encoder(
            env, self.affine_env.weight, self.affine_env.bias,
            self.affine_unit_basic_stats.weight, self.affine_unit_basic_stats.bias, list(groups),
            [l.weight for l in layers], [l.bias for l in layers], wait=wait)
        return ops.linear(x, self.affine_pre_rnn.weight, self.affine_pre_rnn.bias, relu=True), unit_embedding

    def _recur(self, x_tm, hidden, reset=None):
        """x_tm ``[S, B, H]`` time-major -> y_tm ``[S, B, H]``, new hidden in torch's ``[L, B, H]`` form.

        One ``ops.rnn_sequence`` (i2h GEMM + width-selected recurrence kernel) per layer, as ``nn.GRU(num_layers=L)``
        stacks them: layer k reads layer k-1's output sequence, a view of that layer's state buffer (no copy), so
        autograd chains the backward through layer k's ``dx``.

        ``reset``: None, or ``(slot [S, B] int32, h [K, B, L*H], c [K, B, L*H] | None)`` (``ExperienceBatch.reset_*``): at
        a token with ``slot[t, b] = k >= 0`` every layer's state entering step t is replaced by its ``H``-wide slice of row
        (k, b) of the tables."""
        r = self.rnn
        lstm = self.cell == "lstm"
        H = self.hidden_size
        h0, c0 = hidden if lstm else (hidden, None)
        y, hs, cs = x_tm, [], []
        for k in range(self.num_layers):
            rk = None
            if reset is not None:
                slot, rh, rc = reset
                rk = (slot, rh[:, :, k * H:(k + 1) * H].contiguous(), rc[:, :, k * H:(k + 1) * H].contiguous() if lstm else None)
            y, hn, cn = ops.rnn_sequence(y, *r.layer(k), h0[k], c0[k] if lstm else None, self.cell, rk)
            hs.append(hn)
            cs.append(cn)
        h_n = ops.stack_layers(hs)
        return y, ((h_n, ops.stack_layers(cs)) if lstm else h_n)

    def _head_outputs(self, y, unit_embedding, active=None):
        """The attention projection and ONE packed ``[*, 128]`` tensor-core GEMM for the four small heads + the value head
        (25 + value_heads real rows, zero padding; their logits are column ranges of its output, ``ops.pack_cols``), then the target-unit
        dot products -> (packed output, target-unit logits).

        ``active``: None, or the ``(mask, action)`` target-unit rows ``[..., 40]`` of the PPO loss.  The attention layer and the
        target-unit head then run only on the tokens where either row has an entry set (``encoder_ops.target_unit_rows``):
        the same logits there, zeros on the other rows, which the loss never reads."""
        att_w, att_b = self.affine_unit_attention.weight, self.affine_unit_attention.bias
        attention = ops.linear(y, att_w, att_b) if active is None else None
        H = self.hidden_size
        pad = y.new_zeros(ops.PACK_WIDTH - 25 - self.value_heads, H)
        w_pack = torch.cat([self.affine_head_enum.weight, self.affine_move_x.weight, self.affine_move_y.weight,
                            self.affine_head_ability.weight, self.affine_value.weight, pad], dim=0)
        b_pack = torch.cat([self.affine_head_enum.bias, self.affine_move_x.bias, self.affine_move_y.bias,
                            self.affine_head_ability.bias, self.affine_value.bias, pad[:, 0]], dim=0)
        packed = ops.linear(y, w_pack, b_pack)
        if active is None:
            return packed, encoder_ops.target_unit(attention, unit_embedding)
        return packed, encoder_ops.target_unit_rows(y, att_w, att_b, unit_embedding, *encoder_ops.target_rows(*active))

    def _heads(self, y, unit_embedding):
        """Action heads + value (``policy.py:144-155``): column ranges of the packed output, and the target-unit logits."""
        packed, target_unit = self._head_outputs(y, unit_embedding)
        cols = ops.pack_cols(self.value_heads)
        head_enum, move_x, move_y, ability, value = (packed[..., cols[k][0]:cols[k][1]]
                                                     for k in ("enum", "x", "y", "ability", "value"))
        return {'enum': head_enum, 'x': move_x, 'y': move_y, 'target_unit': target_unit, 'ability': ability}, value

    def _run(self, obs, hidden, time_major):
        if not obs[0].is_cuda:
            raise RuntimeError("dotaclient_b200.Policy runs on CUDA only (no CPU fallback); move inputs to cuda")
        x, unit_embedding = self._encode(obs[0], obs[1:])
        x_tm = x if time_major else x.transpose(0, 1)
        y_tm, new_hidden = self._recur(x_tm.contiguous(), hidden)
        y = y_tm if time_major else y_tm.transpose(0, 1)
        logits, value = self._heads(y, unit_embedding)
        return logits, value, new_hidden

    # ------------------------------------------------------------------ class helpers (actor side of the API)
    @classmethod
    def masked_softmax(cls, logits, mask, dim=2):
        """Log-probs normalised over ``mask`` only, no max-subtraction (``policy.py:169-178``).
        The optimizer's hot loop uses the fused kernel instead; this is the API-compatible form."""
        masked_exp = torch.exp(logits).masked_fill(~mask.bool(), 0.)
        return logits - torch.log(masked_exp.sum(dim, keepdim=True))

    @classmethod
    def flatten_selections(cls, inputs):
        """One-hot rows per head from an ``{head: index}`` dict (``policy.py:180-188``)."""
        out = {}
        for key, count in cls.ACTION_OUTPUT_COUNTS.items():
            row = torch.zeros(count, dtype=torch.bool)
            if key in inputs:
                row[inputs[key]] = True
            out[key] = row
        return out

    @classmethod
    def sample_action(cls, logits, mask):
        log_probs = cls.masked_softmax(logits=logits, mask=mask)
        return MaskedCategorical(log_probs=log_probs, mask=mask).sample()     # policy.py:190-195

    @classmethod
    def select_actions(cls, heads_logits, masks):
        """Hierarchical sampling: enum first, then the sub-head it implies (``policy.py:197-216``)."""
        chosen = {'enum': cls.sample_action(heads_logits['enum'], mask=masks['enum'])}
        kind = int(chosen['enum'])
        follow = {1: ('x', 'y'), 2: ('target_unit',), 3: ('ability',)}.get(kind, ())
        for key in follow:
            chosen[key] = cls.sample_action(heads_logits[key], mask=masks[key])
        return chosen

    @classmethod
    def select_actions_batched(cls, heads_logits, masks, u=None):
        """``select_actions`` for a whole pool of agents in ONE kernel launch (``csrc/actor.cu``): ``heads_logits`` /
        ``masks`` are ``{head: [A, n]}`` CUDA tensors (``[A, 1, n]`` accepted), ``u`` optional ``[A, 5]`` uniforms (drawn with
        ``torch.rand`` if omitted).  Returns ``({head: int32 [A]} with -1 where the head was not sampled, logp [A, 5])``.  The picks
        are ``oracle.ref_policy.sample_index``'s up to fp32 rounding near a cumulative boundary (see ``act_batched``)."""
        A = heads_logits['enum'].shape[0]
        dev = heads_logits['enum'].device
        if u is None:
            u = torch.rand(A, 5, device=dev)
        chosen, logp = ops.select_actions([heads_logits[k] for k in ops.HEAD_KEYS], [masks[k] for k in ops.HEAD_KEYS], u.to(dev))
        return {k: chosen[:, h] for h, k in enumerate(ops.HEAD_KEYS)}, logp

    def act_batched(self, hidden, observations, masks, u=None):
        """One environment step for a POOL of ``A`` agents in one pass (the actor side of ``agent.py:578-674`` for many agents
        at once; SURVEY.md 8(f)4): ``Policy.single`` for every agent as ONE ``[1, A]`` time-major forward -- batch-``A``
        recurrence and heads on the same kernels as the optimizer -- followed by the hierarchical masked sampling kernel
        (``select_actions_batched``, one launch for the pool).

        ``hidden``: ``[L, A, H]`` (``(h, c)`` for the LSTM; L = ``num_layers``); ``observations``: ``{key: [A, ...]}`` (what ``single`` takes, with
        a leading agent dimension); ``masks``: ``{head: [A, n]}`` legal-action masks (``action_masks``); ``u``: optional
        ``[A, 5]`` uniforms.  Returns ``(chosen {head: int32 [A], -1 = not sampled}, logp [A, 5], logits {head: [A, n]},
        value [A] ([A, K] with K = value_heads > 1), new hidden)``.  Index selection is ``oracle.ref_policy.sample_index``'s inverse CDF up to fp32 rounding: the two
        agree unless u lies within the rounding band of a cumulative boundary (a few 1e-6 for logits of order 1, up to about
        5e-5 at |logit| 60), where either may take the adjacent legal index.

        Row ``a`` of ``logp`` (log-probability of each sampled head in ``ops.HEAD_KEYS`` order, 0 for heads not sampled) is
        the ``behaviour_logp`` row of this step in agent ``a``'s rollout: what ``DotaOptimizer(advantage_estimator='vtrace')``
        needs to correct for the weights the agent played with."""
        with torch.no_grad():
            obs = {k: v.unsqueeze(0) for k, v in observations.items()}              # [1 (time), A, ...]
            logits, value, new_hidden = self.forward_time_major(obs, hidden)
            flat = {k: v[0] for k, v in logits.items()}
            chosen, logp = self.select_actions_batched(flat, masks, u)
        return chosen, logp, flat, value[0, :, 0] if self.value_heads == 1 else value[0], new_hidden

    @classmethod
    def head_masks(cls, selections):
        """All-ones mask for heads that were used, zeros otherwise (``policy.py:218-224``)."""
        return {key: (torch.ones if key in selections else torch.zeros)(1, 1, n, dtype=torch.bool)
                for key, n in cls.ACTION_OUTPUT_COUNTS.items()}

    @staticmethod
    def ability_available(ability):
        return ability.is_activated and ability.level > 0 and ability.cooldown_remaining == 0 \
            and ability.is_fully_castable                                      # policy.py:226-229

    @classmethod
    def action_masks(cls, player_unit, unit_handles):
        """Legal-action masks for one step (``policy.py:231-260``)."""
        counts = cls.ACTION_OUTPUT_COUNTS
        if not player_unit.is_alive:      # a dead hero can only no-op
            masks = {k: torch.zeros(1, 1, n, dtype=torch.bool) for k, n in counts.items()}
            masks['enum'][0, 0, 0] = True
            return masks
        masks = {k: torch.ones(1, 1, n, dtype=torch.bool) for k, n in counts.items()}
        for ability in player_unit.abilities:
            if ability.slot < 3 and not cls.ability_available(ability):
                masks['ability'][0, 0, ability.slot] = False
        if not masks['ability'].any():
            masks['enum'][0, 0, 3] = False
        valid_units = torch.as_tensor(unit_handles != -1).clone()
        valid_units[0] = False            # the own hero is never a target
        if not valid_units.any():
            masks['enum'][0, 0, 2] = False
        masks['target_unit'][0, 0] = valid_units
        return masks


def fold_value_heads(state_dict):
    """A copy of ``state_dict`` whose K-row value head is folded into the reference's one-row head: W = sum_k W_k and
    b = sum_k b_k, summed in fp32 in head order.  Its value is sum_k V_k, which is the value of the total reward only when
    every head has the same discount.  A one-row head is returned unchanged."""
    out = dict(state_dict)
    w, b = out['affine_value.weight'], out['affine_value.bias']
    if w.shape[0] == 1:
        return out
    ws, bs = w[0].clone(), b[0:1].clone()
    for k in range(1, w.shape[0]):
        ws = ws + w[k]
        bs = bs + b[k:k + 1]
    out['affine_value.weight'], out['affine_value.bias'] = ws.unsqueeze(0), bs
    return out


def split_value_head(state_dict, K):
    """A copy of ``state_dict`` whose one-row value head is split into ``K`` rows of W / K and b / K, so that the summed
    value sum_k V_k starts where the one-row head's value was (up to fp32 rounding of the division)."""
    out = dict(state_dict)
    w, b = out['affine_value.weight'], out['affine_value.bias']
    if w.shape[0] != 1:
        raise ValueError("split_value_head needs a one-row value head, got %s" % (tuple(w.shape),))
    out['affine_value.weight'] = (w / K).expand(K, -1).clone()
    out['affine_value.bias'] = (b / K).expand(K).clone()
    return out
