"""Deterministic synthetic rollouts in the reference's experience wire layout.

Layout = what ``agent.py:350-416`` packs and ``optimizer.py:314-336`` consumes: a dict with
``observations`` (7 fp32 tensors ``[L, units, feat]``), ``masks`` / ``actions`` (5 tensors
``[L, n]``; one-hot or all-zero rows), ``rewards`` (``np.float32 [L, 10]``), plus ids.

Masks and actions are ``torch.bool``: the agent's uint8 masks no longer index under
torch >= 2 (``policy.py:174``), see DESIGN.md "drift".  Distributions follow SURVEY.md 8(d).
"""
import numpy as np
import torch

OBS_SHAPES = {
    "env": (3,),
    "allied_heroes": (1, 12),
    "enemy_heroes": (5, 12),
    "allied_nonheroes": (16, 12),
    "enemy_nonheroes": (16, 12),
    "allied_towers": (1, 12),
    "enemy_towers": (1, 12),
}
HEAD_SIZES = {"enum": 4, "x": 9, "y": 9, "target_unit": 40, "ability": 3}


def make_rollout(length, seed, game_id=0, team_id=2, weight_version=1, with_canvas=False):
    """One rollout of ``length`` steps.  ``seed`` fully determines it (CPU generator)."""
    g = torch.Generator().manual_seed(int(seed))
    L = int(length)
    obs = {k: torch.randn((L,) + shp, generator=g, dtype=torch.float32) for k, shp in OBS_SHAPES.items()}
    rewards = (torch.randn((L, 10), generator=g, dtype=torch.float32) * 0.01).numpy()
    enum = torch.randint(0, 4, (L,), generator=g)
    masks = {k: torch.zeros((L, n), dtype=torch.bool) for k, n in HEAD_SIZES.items()}
    actions = {k: torch.zeros((L, n), dtype=torch.bool) for k, n in HEAD_SIZES.items()}
    rows = torch.arange(L)
    masks["enum"][:] = True
    actions["enum"][rows, enum] = True
    move, attack, ability = enum == 1, enum == 2, enum == 3
    for k in ("x", "y"):
        pick = torch.randint(0, 9, (L,), generator=g)
        masks[k][move] = True
        actions[k][rows[move], pick[move]] = True
    valid = torch.rand((L, 40), generator=g) < 0.5
    valid[:, 0] = False                                   # the own hero is never a target (policy.py:255)
    forced = torch.randint(1, 40, (L,), generator=g)
    valid[rows, forced] = True                            # at least one valid unit
    score = torch.rand((L, 40), generator=g).masked_fill(~valid, -1.0)
    target = score.argmax(dim=1)                          # uniform over the valid units
    masks["target_unit"][attack] = valid[attack]
    actions["target_unit"][rows[attack], target[attack]] = True
    pick = torch.randint(0, 3, (L,), generator=g)
    masks["ability"][ability] = True
    actions["ability"][rows[ability], pick[ability]] = True
    data = {
        "game_id": game_id, "team_id": team_id, "player_id": 0, "weight_version": weight_version,
        "observations": obs, "masks": masks, "actions": actions, "rewards": rewards,
    }
    if with_canvas:
        data["canvas"] = np.zeros((256, 256, 3), dtype=np.uint8)   # agent.py:424-437
    return data


def demonstration_rollout(policy, length, seed, game_id=0, team_id=2, weight_version=1):
    """``make_rollout(length, seed, ...)`` with the actions a demonstrator picked: ``policy`` (a ``Policy`` on a CUDA
    device) plays every step with ``act_batched``, from its zero state, over the rollout's own observations, open loop (its
    actions do not change the observations), with uniforms drawn from a generator that ``seed`` fixes.  The legal actions
    of a step are every enum, x, y and ability entry and a seeded set of at least one target unit (never unit 0).  As an
    agent stores them, the step's ``masks`` hold the enum row and the legal rows of the heads the enum action sampled, and
    the other heads' rows are zero."""
    from dotaclient_b200.ops import HEAD_KEYS
    data = make_rollout(length, seed, game_id=game_id, team_id=team_id, weight_version=weight_version)
    L = int(length)
    g = torch.Generator().manual_seed(int(seed) + 104729)
    units = torch.rand((L, 40), generator=g) < 0.5
    units[:, 0] = False
    units[torch.arange(L), torch.randint(1, 40, (L,), generator=g)] = True
    u = torch.rand((L, 5), generator=g)
    legal = {k: torch.ones((L, n), dtype=torch.bool) for k, n in HEAD_SIZES.items()}
    legal["target_unit"] = units
    dev = next(policy.parameters()).device
    hidden = policy.init_hidden()
    hidden = tuple(x.to(dev) for x in hidden) if isinstance(hidden, tuple) else hidden.to(dev)
    picks = []
    for t in range(L):
        chosen, _, _, _, hidden = policy.act_batched(hidden, {k: v[t:t + 1].to(dev) for k, v in data["observations"].items()},
                                                     {k: legal[k][t:t + 1].to(dev) for k in HEAD_KEYS}, u[t:t + 1].to(dev))
        picks.append(torch.stack([chosen[k] for k in HEAD_KEYS], dim=1))
    picks = torch.cat(picks).long().cpu()                 # [L, 5], -1 where the head was not sampled
    for h, k in enumerate(HEAD_KEYS):
        rows = picks[:, h] >= 0
        data["masks"][k] = torch.where(rows[:, None], legal[k], torch.zeros_like(legal[k]))
        act = torch.zeros((L, HEAD_SIZES[k]), dtype=torch.bool)
        act[torch.nonzero(rows).flatten(), picks[rows, h]] = True
        data["actions"][k] = act
    return data


def split_rollout(data, cuts, initial_hiddens=None):
    """One game's rollout -> the pieces an actor publishing every few steps sends: cut before each step in ``cuts``
    (increasing, each in ``[1, L)``).  Piece p holds steps ``[a, b)``.  Every piece but the last is ``'terminal': False``
    and its observations carry ``b - a + 1`` rows: row ``b - a`` is the observation after its last step, which is also the
    next piece's row 0.  The last piece is ``'terminal': True``.  ``initial_hiddens`` (optional, one entry per piece, None
    for none) become the pieces' ``'initial_hidden'``: the actor's recurrent state entering the piece's first step."""
    L = int(data['rewards'].shape[0])
    bounds = [0] + [int(c) for c in cuts] + [L]
    if any(b <= a for a, b in zip(bounds, bounds[1:])):
        raise ValueError("cuts=%r: must increase strictly within [1, %d)" % (list(cuts), L))
    if initial_hiddens is not None and len(initial_hiddens) != len(bounds) - 1:
        raise ValueError("initial_hiddens: %d entries for %d pieces" % (len(initial_hiddens), len(bounds) - 1))
    pieces = []
    for p, (a, b) in enumerate(zip(bounds, bounds[1:])):
        last = b == L
        piece = {k: v for k, v in data.items() if k not in ('observations', 'masks', 'actions', 'rewards', 'behaviour_logp')}
        piece['observations'] = {k: v[a:b if last else b + 1] for k, v in data['observations'].items()}
        for k in ('masks', 'actions'):
            piece[k] = {h: v[a:b] for h, v in data[k].items()}
        piece['rewards'] = data['rewards'][a:b]
        if 'behaviour_logp' in data:
            piece['behaviour_logp'] = data['behaviour_logp'][a:b]
        piece['terminal'] = last
        if initial_hiddens is not None and initial_hiddens[p] is not None:
            piece['initial_hidden'] = initial_hiddens[p]
        pieces.append(piece)
    return pieces


def rollout_seed(rank, index):
    """SURVEY.md 8(d): ``7 + 1000*rank + i``."""
    return 7 + 1000 * int(rank) + int(index)


def ragged_lengths(n, seq_len, seed):
    """Correctness configs: L ~ U[S/2, 3S] so multi-chunk carry and tail padding are exercised."""
    rng = np.random.RandomState(seed)
    return [int(v) for v in rng.randint(max(1, seq_len // 2), 3 * seq_len + 1, size=n)]
