"""The callers either side of the self-play path, in bulk (SURVEY.md 8f-2 / 8f-3).

* ``Reanalyse`` - same constructor and ``reanalyse(replay_buffer, shared_storage)`` loop as the reference actor
  (``replay_buffer.py:307-373``), but the fresh root values of MANY games come from ONE call per batch (the
  representation + prediction kernels of the search path, with ``support_to_scalar`` fused behind the value head)
  instead of one game per RPC on the CPU: ``mz_reanalyse_values``, which stacks the observations on the GPU, for
  configs with stacked observations, chunked ``mz_initial_inference`` otherwise.  With ``config.reanalyse_search`` the
  self-play search is also re-run at every position (``mz_reanalyse_search``, the MuZero paper's Reanalyze) and its
  visit distribution replaces the game's ``child_visits``, the policy targets.
* ``initial_priorities`` / ``save_games`` - the prioritised-replay priorities ``ReplayBuffer.save_game`` computes one
  position at a time in Python (``replay_buffer.py:33-51`` calling ``compute_target_value``, ``:230-262``), evaluated
  for a whole game with array arithmetic in the reference's operation order (bit-identical float32 priorities), and
  attached before the game is handed over, so the unmodified ``save_game`` skips its loop
  (``if game_history.priorities is not None``).

Nothing here imports torch; the engine does the arithmetic on the GPU.
"""
from __future__ import annotations

import itertools
import time

import numpy

from .engine import SearchEngine


def _call(obj, method, *args, **kw):
    fn = getattr(obj, method)
    if hasattr(fn, "remote"):
        import ray
        return ray.get(fn.remote(*args, **kw))
    return fn(*args, **kw)


def _fire(obj, method, *args):
    fn = getattr(obj, method)
    return fn.remote(*args) if hasattr(fn, "remote") else fn(*args)


def _frame_source(gh):
    """(frame rows, action history, positions T) of a game without building anything per position: a
    ``PackedGameHistory`` whose lists were never built gives its block's contiguous ``obs`` [T + 1][O] float32 and
    ``action`` sections, any other history its ``observation_history`` list (rows converted when read) and
    ``action_history``."""
    d = getattr(gh, "__dict__", {})
    if "_packed" in d and "observation_history" not in d:
        g = d["_packed"][0]
        T = int(g["length"])
        actions = numpy.empty(T + 1, numpy.int32)
        actions[0] = 0
        actions[1:] = g["action"]
        return numpy.asarray(g["obs"], dtype=numpy.float32).reshape(T + 1, -1), actions, T
    return gh.observation_history, gh.action_history, len(gh.root_values)


def _to_play(gh, T):
    """``to_play_history[:T]`` as int32, read from a ``PackedGameHistory``'s block without building its lists."""
    d = getattr(gh, "__dict__", {})
    if "_packed" in d and "to_play_history" not in d:
        g = d["_packed"][0]
        return numpy.concatenate([[int(g["first_to_play"])], numpy.asarray(g["to_play"]).reshape(-1)])[:T].astype(numpy.int32)
    return numpy.asarray(gh.to_play_history[:T], dtype=numpy.int32).reshape(T)


def policy_rows(visit_counts, legal_mask, action_space):
    """The ``child_visits`` rows ``GameHistory.store_visit_counts`` builds from a search's visit counts [T][A] and the
    legal masks [T][A]: ``visit / total`` for legal actions, ``0`` for the others."""
    rows = []
    for visits, legal in zip(visit_counts, legal_mask):
        total = int(visits.sum())
        rows.append([int(visits[a]) / total if legal[a] else 0 for a in action_space])
    return rows


def _row(rows, i):
    """Frame i of a source as float32 [O]: ``numpy.asarray(get_stacked_observations(i, 0, A), float32)`` flattened."""
    return numpy.asarray(rows[i], dtype=numpy.float32).reshape(-1)


def pack_frames(sources):
    """The arguments of ``SearchEngine.reanalyse_values`` for ``_frame_source`` tuples: every game's frames once as
    float32 [sum (T + 1)][O] (O(T * O) host memory, no stack) and its action history as int32, back to back, with the
    per-game offsets and positions."""
    O = next(_row(rows, 0).size for rows, _, T in sources if T)
    frame_off = numpy.zeros(len(sources) + 1, numpy.int64)
    action_off = numpy.zeros(len(sources) + 1, numpy.int64)
    for g, (rows, actions, _) in enumerate(sources):
        frame_off[g + 1] = frame_off[g] + len(rows)
        action_off[g + 1] = action_off[g] + len(actions)
    frames = numpy.empty((int(frame_off[-1]), O), numpy.float32)
    for g, (rows, _, _) in enumerate(sources):
        if isinstance(rows, numpy.ndarray):
            frames[frame_off[g]:frame_off[g + 1]] = rows.reshape(len(rows), O)
        else:                                            # one row at a time: no second copy of the game
            for k in range(len(rows)):
                frames[frame_off[g] + k] = _row(rows, k)
    actions = numpy.concatenate([numpy.asarray(a, dtype=numpy.int32).reshape(-1) for _, a, _ in sources])
    positions = numpy.array([T for _, _, T in sources], numpy.int64)
    return dict(frames=frames, frame_offsets=frame_off, actions=actions, action_offsets=action_off, positions=positions)


class _Batch:
    """The games of one Reanalyse call: their ``_frame_source`` tuples, packed by ``pack_frames`` at most once."""

    def __init__(self, game_histories):
        self.sources = [_frame_source(gh) for gh in game_histories]
        self.counts = [T for _, _, T in self.sources]
        self._packed = None

    @property
    def packed(self):
        if self._packed is None:
            self._packed = pack_frames(self.sources)
        return self._packed


class Reanalyse:
    """Updates games of the replay buffer with fresh value estimates (MuZero paper, appendix Reanalyse) and, with
    ``config.reanalyse_search``, fresh policy targets from a new search at every position."""

    # A reanalysed game is searched under game id SEARCH_GAME_IDS + its replay-buffer id (training games are numbered
    # from 0, test games from SelfPlay.TEST_GAME_IDS = 1 << 40).  The search's Philox streams key a game by the low 32
    # bits of its id, so the id alone does not keep them apart from self-play's: the search handle's seed does.  It is
    # config.seed with SEARCH_SEED_XOR in its high word, which puts the Philox key's high word outside that of every
    # self-play seed (config.seed + worker index), so no noise or tie-break of a reanalysis repeats a self-play draw.
    SEARCH_GAME_IDS = 1 << 41
    SEARCH_SEED_XOR = 0x7169E0A5 << 32

    def __init__(self, initial_checkpoint, config, device=0, max_positions=None, games_per_call=None, Game=None):
        self.config = config
        self.Game = Game
        numpy.random.seed(config.seed)                     # replay_buffer.py:318
        self.max_positions = int(max_positions or getattr(config, "reanalyse_max_positions", 4096))
        self.games_per_call = int(games_per_call or getattr(config, "reanalyse_games_per_call", 64))
        searching = bool(getattr(config, "reanalyse_search", False))
        if searching and not callable(getattr(Game, "legal_masks", None)):
            raise ValueError("config.reanalyse_search needs the game plug-in's Game.legal_masks(observations) hook (the "
                             "legal mask of each raw frame; a GameHistory does not store legal actions): pass Game= a "
                             "plug-in class that has it")
        # inference only: num_simulations = 0 keeps the node / hidden-state pools at one entry per position
        self.engine = SearchEngine(config, max_games=self.max_positions, device=device, num_simulations=0)
        self.engine.load_weights(initial_checkpoint["weights"])
        # The search runs on a handle of its own: a search whose x3 towers leave the fp16 range switches its handle to the
        # fp32 towers for good, and the values must not depend on whether a search ran before them.
        self.search_engine = None
        if searching:
            self.search_engine = SearchEngine(config, max_games=self.max_positions, device=device,
                                              seed=self.search_seed(config.seed),
                                              num_simulations=int(config.num_simulations))
            self.search_engine.load_weights(initial_checkpoint["weights"])
        self.num_reanalysed_games = initial_checkpoint.get("num_reanalysed_games", 0)

    @classmethod
    def search_seed(cls, seed):
        """The seed of the search handle for a config seed (see SEARCH_SEED_XOR)."""
        return (int(seed) ^ cls.SEARCH_SEED_XOR) & 0xFFFFFFFFFFFFFFFF

    def set_weights(self, weights):
        self.engine.load_weights(weights)
        if self.search_engine is not None:
            self.search_engine.load_weights(weights)

    def close(self):
        self.engine.close()
        if self.search_engine is not None:
            self.search_engine.close()

    # ------------------------------------------------------------------ the batched core
    def fresh_root_values(self, game_histories):
        """``models.support_to_scalar(model.initial_inference(observations)[0])`` (replay_buffer.py:345-366) for every
        position of every game, batched over games; returns one float32 array per game (``torch.squeeze`` shape:
        ``[T]``, or 0-d for a one-position game).

        With ``stacked_observations`` s > 0 the host hands each game's frames over once and the stacked inputs are built
        on the GPU (``SearchEngine.reanalyse_values``); with s = 0 the observations are gathered one chunk of
        ``max_positions`` at a time for ``initial_inference``.  Either way no per-position stack is built on the host."""
        return self._root_values(_Batch(game_histories))

    def _root_values(self, batch):
        counts = batch.counts
        total = sum(counts)
        if not total:
            return [numpy.zeros(0, numpy.float32) for _ in counts]
        if int(self.config.stacked_observations) > 0:
            p = batch.packed
            values = self.engine.reanalyse_values(p["frames"], p["frame_offsets"], p["actions"], p["action_offsets"],
                                                  p["positions"])
        else:
            values = self._plain_values(batch.sources, total)
        out, off = [], 0
        for T in counts:
            v = values[off:off + T].copy()
            out.append(v.reshape(()) if T == 1 else v)
            off += T
        return out

    def _plain_values(self, sources, total):
        """s = 0: the observation of each position is its frame; one initial_inference per max_positions positions."""
        values = numpy.empty(total, numpy.float32)
        flat = ((rows, i) for rows, _, T in sources for i in range(T))
        for lo in range(0, total, self.max_positions):
            hi = min(total, lo + self.max_positions)
            obs = numpy.stack([_row(rows, i) for rows, i in itertools.islice(flat, hi - lo)])
            values[lo:hi] = self.engine.initial_inference(obs)["value"]
        return values

    def fresh_search(self, game_histories, game_ids):
        """``MCTS.run(model, gh.get_stacked_observations(i, s, A), legal_actions_i, gh.to_play_history[i], True)`` at
        every position i of every game, batched over games (one ``SearchEngine.reanalyse_search``, chunks of
        ``max_positions`` positions) on the search handle (seed ``search_seed(config.seed)``); game g is searched
        under game id ``SEARCH_GAME_IDS + game_ids[g]`` and move index i.  The legal actions come from the plug-in's
        ``Game.legal_masks`` on the game's frames.  Returns one (visit_counts int32 [T][A], root_values float64 [T],
        legal_mask uint8 [T][A]) per game."""
        return self._search(_Batch(game_histories), game_histories, game_ids)

    def _search(self, batch, game_histories, game_ids):
        A = len(self.config.action_space)
        counts = batch.counts
        if not sum(counts):
            return [(numpy.zeros((0, A), numpy.int32), numpy.zeros(0), numpy.zeros((0, A), numpy.uint8))
                    for _ in game_histories]
        p = batch.packed
        shape = tuple(self.config.observation_shape)
        fo = p["frame_offsets"]
        legal = numpy.concatenate([
            numpy.asarray(self.Game.legal_masks(p["frames"][fo[g]:fo[g] + T].reshape((T,) + shape)),
                          dtype=numpy.uint8).reshape(T, A)
            for g, T in enumerate(counts) if T])
        to_play = numpy.concatenate([_to_play(gh, T) for gh, T in zip(game_histories, counts)])
        ids = self.SEARCH_GAME_IDS + numpy.asarray(list(game_ids), dtype=numpy.int64)
        visits, root = self.search_engine.reanalyse_search(p["frames"], fo, p["actions"], p["action_offsets"],
                                                           p["positions"], legal, to_play, ids,
                                                           add_exploration_noise=True)
        out, off = [], 0
        for T in counts:
            out.append((visits[off:off + T], root[off:off + T], legal[off:off + T]))
            off += T
        return out

    def reanalyse_games(self, game_histories, game_ids=None):
        """Set ``reanalysed_predicted_root_values`` on every history (one batched inference) and, with
        ``config.reanalyse_search``, replace every position's ``child_visits`` row with that of a fresh search
        (``fresh_search``; ``game_ids`` are the games' replay-buffer ids, 0 .. n - 1 when not given); returns the
        histories.  The games' frames are packed for the library once, for both calls."""
        batch = _Batch(game_histories)
        if self.config.use_last_model_value:
            for gh, v in zip(game_histories, self._root_values(batch)):
                gh.reanalysed_predicted_root_values = v
        if self.search_engine is not None:
            ids = range(len(game_histories)) if game_ids is None else game_ids
            action_space = self.config.action_space
            for gh, (visits, _, legal) in zip(game_histories, self._search(batch, game_histories, ids)):
                gh.child_visits = policy_rows(visits, legal, action_space)
        self.num_reanalysed_games += len(game_histories)
        return game_histories

    # ------------------------------------------------------------------ the reference's actor loop
    def reanalyse(self, replay_buffer, shared_storage):
        cfg = self.config
        while _call(shared_storage, "get_info", "num_played_games") < 1:
            time.sleep(0.1)
        while (_call(shared_storage, "get_info", "training_step") < cfg.training_steps
               and not _call(shared_storage, "get_info", "terminate")):
            self.set_weights(_call(shared_storage, "get_info", "weights"))
            sampled = [_call(replay_buffer, "sample_game", force_uniform=True) for _ in range(self.games_per_call)]
            games = {}
            for game_id, game_history, _ in sampled:       # the same game may be drawn twice: analyse it once
                games.setdefault(game_id, game_history)
            self.reanalyse_games(list(games.values()), list(games.keys()))
            for game_id, game_history in games.items():
                _fire(replay_buffer, "update_game_history", game_id, game_history)
            _fire(shared_storage, "set_info", "num_reanalysed_games", self.num_reanalysed_games)


# ----------------------------------------------------------------------------------------------------------------
# bulk ingest: PER priorities of whole games
# ----------------------------------------------------------------------------------------------------------------
def _weak_scalar_dtype(dtype):
    """dtype of ``dtype.type(1) * 1.0``: float32 under NumPy >= 2 (NEP 50, Python floats are weak), float64 under the
    value-based casting of the NumPy 1.21 the reference pins - whichever the installed NumPy does, the reference's
    scalar arithmetic on ``reanalysed_predicted_root_values`` (a float32 array) does the same."""
    return (numpy.dtype(dtype).type(1) * 1.0).dtype


def target_values(game_history, config):
    """``ReplayBuffer.compute_target_value`` (replay_buffer.py:230-262) for every position of a game at once.

    The reference starts from ``last_step_value * discount**td_steps`` (or the int 0 when the bootstrap index is past the
    end) and adds the signed rewards ``reward * discount**i`` for i = 0, 1, ... in that order; the same additions happen
    here in the same order and in the same floating-point type, element-wise over all positions, so every value is
    bit-identical to the scalar loop.  Returns a list of numpy scalars (float64, or float32 where the reference's own
    arithmetic stays in float32 because the bootstrap value comes from a float32 array)."""
    T = len(game_history.root_values)
    td, discount = int(config.td_steps), config.discount
    reanalysed = game_history.reanalysed_predicted_root_values is not None
    src = game_history.reanalysed_predicted_root_values if reanalysed else game_history.root_values
    if reanalysed:
        roots = numpy.asarray(src).reshape(-1)
        boot_dtype = _weak_scalar_dtype(roots.dtype)
    else:
        roots = numpy.asarray([0.0 if r is None else r for r in src], dtype=numpy.float64)
        boot_dtype = numpy.dtype(numpy.float64)
    to_play = numpy.asarray(game_history.to_play_history, dtype=numpy.int64)
    rewards = numpy.asarray(game_history.reward_history, dtype=numpy.float64)
    idx = numpy.arange(T)
    boot = idx + td
    has = boot < T
    acc = numpy.zeros(T, boot_dtype)                     # positions WITH a bootstrap value: its dtype rules
    plain = numpy.zeros(T, numpy.float64)                # positions without: Python-float arithmetic
    if has.any():
        b = boot[has]
        last = numpy.where(to_play[b] == to_play[idx[has]], roots[b], -roots[b]).astype(roots.dtype)
        acc[has] = (last * discount ** td).astype(boot_dtype)
    n_hist = len(rewards)
    for i in range(td):
        j = idx + 1 + i                                  # reward_history[index + 1 + i], while inside [index+1, bootstrap]
        ok = j < n_hist
        if not ok.any():
            break
        jj = numpy.where(ok, j, 0)
        same = to_play[idx] == to_play[numpy.minimum(idx + i, len(to_play) - 1)]
        term = numpy.where(same, rewards[jj], -rewards[jj]) * discount ** i
        plain = numpy.where(ok, plain + term, plain)
        acc = numpy.where(ok, acc + term.astype(boot_dtype), acc)       # a weak Python float joins in acc's own type
    return [acc[i] if has[i] else plain[i] for i in range(T)]


def initial_priorities(game_history, config):
    """The ``priorities`` array and ``game_priority`` that ``save_game`` would compute (replay_buffer.py:39-51)."""
    tv = target_values(game_history, config)
    alpha = config.PER_alpha
    pri = [numpy.abs(root_value - tv[i]) ** alpha for i, root_value in enumerate(game_history.root_values)]
    pri = numpy.array(pri, dtype="float32")
    return pri, numpy.max(pri)


def save_games(replay_buffer, game_histories, config, shared_storage=None):
    """Hand a batch of finished games to an (unmodified) ``ReplayBuffer``: priorities are attached first, so its
    per-position Python loop is skipped; every other effect of ``save_game`` (eviction, counters) is the reference's."""
    for gh in game_histories:
        if config.PER and gh.priorities is None:
            gh.priorities, gh.game_priority = initial_priorities(gh, config)
        _fire(replay_buffer, "save_game", gh, shared_storage)
