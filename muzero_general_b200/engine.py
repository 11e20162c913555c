"""Python face of the C ABI: one ``SearchEngine`` per GPU process.

``SearchEngine`` owns an ``MzHandle`` and exposes, for a whole batch of games,
what the reference does for one game at a time:

* ``load_weights(state_dict)``          <- ``model.set_weights`` (models.py:72-73)
* ``search(...)``                       <- ``MCTS(config).run`` (self_play.py:260-361)
* ``initial_inference / recurrent_inference``  (models.py:172-195, 601-623)
* ``export_tree(game)``                 <- walking ``Node.children`` (self_play.py:433-449)

All numerical work happens in libmzb200.so; this file only marshals buffers.  Inputs may be
numpy arrays (host memory, copies are part of the call) or CUDA torch tensors (device memory).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Optional

import numpy

from . import _lib
from .netspec import FC, NetSpec, netspec_from_config, weights_spec


def _is_torch(x):
    return x is not None and type(x).__module__.startswith("torch")


def _fill_layers(desc, prefix, layers):
    if len(layers) > _lib.MZ_MAX_LAYERS:
        raise ValueError(f"at most {_lib.MZ_MAX_LAYERS} hidden layers per head are supported")
    setattr(desc, "n_" + prefix, len(layers))
    arr = getattr(desc, prefix)
    for i, v in enumerate(layers):
        arr[i] = int(v)


def net_desc(spec: NetSpec) -> _lib.MzNetDesc:
    d = _lib.MzNetDesc()
    d.kind = spec.kind
    d.obs_c, d.obs_h, d.obs_w = spec.in_channels, spec.obs_shape[1], spec.obs_shape[2]
    d.action_space = spec.action_space
    d.support_size = spec.support_size
    d.encoding = spec.encoding
    _fill_layers(d, "fc_representation", spec.fc_representation)
    _fill_layers(d, "fc_dynamics", spec.fc_dynamics)
    _fill_layers(d, "fc_reward", spec.fc_reward)
    _fill_layers(d, "fc_value", spec.fc_value)
    _fill_layers(d, "fc_policy", spec.fc_policy)
    d.blocks, d.channels = spec.blocks, spec.channels
    d.reduced_reward, d.reduced_value, d.reduced_policy = spec.reduced_reward, spec.reduced_value, spec.reduced_policy
    _fill_layers(d, "res_fc_reward", spec.res_fc_reward)
    _fill_layers(d, "res_fc_value", spec.res_fc_value)
    _fill_layers(d, "res_fc_policy", spec.res_fc_policy)
    d.downsample = spec.downsample
    return d


@dataclass
class SearchOutput:
    visit_counts: numpy.ndarray          # [n, A] int32
    root_value: numpy.ndarray            # [n] float64
    root_predicted_value: numpy.ndarray  # [n] float32
    max_tree_depth: numpy.ndarray        # [n] int32
    tie_count: numpy.ndarray             # [n] int32
    root_priors: numpy.ndarray           # [n, A] float64
    value_range: numpy.ndarray           # [n, 2] float64
    trace: Optional[dict] = None
    device_ms: float = 0.0


# SearchOutput's arrays in field order: (dtype, columns per game: 0 = one value, -1 = one per action)
_OUT_FIELDS = (("int32", -1), ("float64", 0), ("float32", 0), ("int32", 0), ("int32", 0), ("float64", -1), ("float64", 2))


def output_layout(n, A):
    """Where a device-memory search puts SearchOutput's seven arrays in the one buffer it allocates for them: per field
    (dtype, shape, strides, byte offset), offsets 16-byte aligned, and the buffer's size in bytes (a multiple of 16)."""
    fields, off = [], 0
    for dt, cols in _OUT_FIELDS:
        shape = (n,) if cols == 0 else (n, A if cols < 0 else cols)
        fields.append((dt, shape, (1,) if cols == 0 else (shape[1], 1), off))
        off += (numpy.dtype(dt).itemsize * math.prod(shape) + 15) & ~15
    return tuple(fields), off


def carve_outputs(buf, fields):
    """SearchOutput whose arrays are views of ``buf``, a float64 torch tensor of output_layout's size."""
    import torch
    views = {"float64": buf, "float32": buf.view(torch.float32), "int32": buf.view(torch.int32)}
    return SearchOutput(*[views[dt].as_strided(shape, strides, off // (8 if dt == "float64" else 4))
                          for dt, shape, strides, off in fields])


_TORCH_DTYPES = {}


class SearchEngine:
    def __init__(self, config, max_games: int = 1, device: int = 0, seed: Optional[int] = None,
                 num_simulations: Optional[int] = None, extra_expansions: int = 0):
        self.lib = _lib.load_library()
        self.config = config
        self.spec = netspec_from_config(config)
        if list(config.action_space) != list(range(len(config.action_space))):
            raise ValueError("action_space must be list(range(n)) (every reference game file is)")
        if list(config.players) != list(range(len(config.players))):
            raise ValueError("players must be list(range(n))")
        self.A = self.spec.action_space
        self.N = int(config.num_simulations if num_simulations is None else num_simulations)
        self.max_games = int(max_games)
        self.device = int(device)
        self.extra_expansions = int(extra_expansions)       # pool room for searches continued from an imported tree
        self.pool_n = self.N + self.extra_expansions
        s = _lib.MzSearchDesc()
        s.max_games = self.max_games
        s.num_simulations = self.N
        s.extra_expansions = self.extra_expansions
        s.num_players = len(config.players)
        s.discount = float(config.discount)
        s.pb_c_base = float(config.pb_c_base)
        s.pb_c_init = float(config.pb_c_init)
        s.root_dirichlet_alpha = float(config.root_dirichlet_alpha)
        s.root_exploration_fraction = float(config.root_exploration_fraction)
        s.seed = int(config.seed if seed is None else seed) & 0xFFFFFFFFFFFFFFFF
        # math.log / math.sqrt exactly as the reference evaluates them (self_play.py:385-390)
        n = self.pool_n + 2
        self._pbc = (C.c_double * n)(*[math.log((i + config.pb_c_base + 1) / config.pb_c_base) + config.pb_c_init
                                       for i in range(n)])
        self._sqrt = (C.c_double * n)(*[math.sqrt(i) for i in range(n)])
        s.pb_c_table = C.cast(self._pbc, C.POINTER(C.c_double))
        s.sqrt_table = C.cast(self._sqrt, C.POINTER(C.c_double))
        # the whole exploration factor pb_c(n_p) * (sqrt(n_p) / (n_c + 1)) with Python's own roundings
        self._ucb = (C.c_double * (n * n))(*[self._pbc[p] * (self._sqrt[p] / (c + 1)) for p in range(n) for c in range(n)])
        s.ucb_table = C.cast(self._ucb, C.POINTER(C.c_double))
        self._net_desc = net_desc(self.spec)
        handle = C.c_void_p()
        rc = self.lib.mz_create(C.byref(self._net_desc), C.byref(s), self.device, C.byref(handle))
        if rc != 0:
            msg = self.lib.mz_last_error(None).decode()
            if rc == _lib.MZ_EUNSUPPORTED:
                raise NotImplementedError(msg)
            raise _lib.MzError(rc, msg)
        self._h = handle
        self.hidden_elems = int(self.lib.mz_hidden_elems(self._h))
        self.obs_elems = int(self.lib.mz_obs_elems(self._h))
        self._dio = _lib.MzDeviceSearchIO()            # one argument struct for every mz_search_device call
        self._dio_ref = C.byref(self._dio)
        self._next_out = None                           # ((n_games, device), (buffer, layout, offsets)) of the next device search

    # ------------------------------------------------------------------ plumbing
    def close(self):
        self._next_out = None
        if getattr(self, "_h", None):
            self.lib.mz_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise _lib.MzError(rc, self.lib.mz_last_error(self._h).decode())

    @property
    def launch_count(self):
        return int(self.lib.mz_launch_count(self._h))

    @property
    def graph_partitions(self):
        """Parallel branches of the replayed search graph (1 = one chain of kernels)."""
        return int(self.lib.mz_graph_partitions(self._h))

    @property
    def last_fc_launch(self):
        """Shape of this handle's last fused FC search launch (grid, block, group, smem, ctas_per_sm), None before one."""
        info = (C.c_int64 * 5)()
        if self.lib.mz_fc_last_launch(self._h, info) != 1:
            return None
        return dict(zip(("grid", "block", "group", "smem", "ctas_per_sm"), (int(v) for v in info)))

    @property
    def fc_prepared(self):
        """The fused FC launch kept for the next search (mz_debug_fc_prepared), None when there is none."""
        info = (C.c_int64 * 7)()
        if self.lib.mz_debug_fc_prepared(self._h, info) != 1:
            return None
        return dict(zip(("games", "group", "threads", "generic", "one_level", "select_levels", "fixed_shape"),
                        (int(v) for v in info)))

    @property
    def last_search_ms(self):
        return float(self.lib.mz_last_search_ms(self._h))

    @property
    def numerics(self):
        """Arithmetic of the search path (bench.py's dtype)."""
        return self.lib.mz_numerics(self._h).decode()

    KERNEL_CLASSES = ("tree_step_kernel", "conv_tower_tc_kernel", "heads_kernel", "conv3x3_kernel", "other", "small_tower_kernel",
                      "small_search_kernel")

    def kernel_timing(self, enable):
        """Bracket every kernel of the step-wise pipeline with CUDA events (no graph replay while enabled)."""
        self._check(self.lib.mz_kernel_timing(self._h, 1 if enable else 0))

    def kernel_times(self):
        """{kernel class: (total ms, launches)} since the last call (mz_kernel_times)."""
        import ctypes as C
        ms = (C.c_double * len(self.KERNEL_CLASSES))()
        cnt = (C.c_int64 * len(self.KERNEL_CLASSES))()
        self._check(self.lib.mz_kernel_times(self._h, ms, cnt))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.KERNEL_CLASSES)}

    @staticmethod
    def _ptr(x, dtype, keep):
        """Pointer of a numpy array (made contiguous, right dtype) or of a CUDA torch tensor."""
        if x is None:
            return None
        if _is_torch(x):
            if not _TORCH_DTYPES:
                import torch
                _TORCH_DTYPES.update({numpy.float32: torch.float32, numpy.float64: torch.float64, numpy.int32: torch.int32,
                                      numpy.int64: torch.int64, numpy.uint8: torch.uint8})
            want = _TORCH_DTYPES[dtype]
            if x.dtype != want or not x.is_contiguous():
                x = x.to(want).contiguous()
            keep.append(x)
            return x.data_ptr()
        a = numpy.ascontiguousarray(x, dtype=dtype)
        keep.append(a)
        return a.ctypes.data

    # ------------------------------------------------------------------ weights
    def load_weights(self, state_dict):
        """Accepts the reference ``state_dict`` (torch tensors or numpy arrays, CPU)."""
        tensors, keep = [], []
        for key, shape in weights_spec(self.spec):
            if key.endswith("num_batches_tracked"):
                continue
            if key not in state_dict:
                raise KeyError(f"state_dict is missing {key}")
            v = state_dict[key]
            if _is_torch(v):
                v = v.detach().cpu().numpy()
            a = numpy.ascontiguousarray(v, dtype=numpy.float32)
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"{key}: expected shape {tuple(shape)}, got {tuple(a.shape)}")
            keep.append(a)
            tensors.append((key.encode(), a))
        arr = (_lib.MzTensor * len(tensors))()
        for i, (name, a) in enumerate(tensors):
            arr[i].name = name
            arr[i].data = a.ctypes.data
            arr[i].numel = a.size
        self._check(self.lib.mz_load_weights(self._h, arr, len(tensors)))

    # ------------------------------------------------------------------ search
    def search(self, obs=None, legal_mask=None, to_play=None, add_exploration_noise=False, noise=None,
               first_index=None, game_id=None, move_index=None, teacher=None, trace=False, trace_depth=None,
               keep_tree=False, stepwise=False, n_games=None, continue_tree=False) -> SearchOutput:
        A, N = self.A, self.N
        keep = []
        if n_games is None:
            src = obs if obs is not None else (teacher["root_value"] if teacher else legal_mask)
            n_games = 1 if (src is None and continue_tree) else int(src.shape[0])
        n = n_games
        device_mem = _is_torch(obs)
        if legal_mask is not None and not _is_torch(legal_mask):
            # the reference asserts this per game (self_play.py:296); a row without a legal action would also
            # index the node pool out of bounds on the device
            assert numpy.asarray(legal_mask).reshape(n, -1).any(axis=1).all(), \
                "Legal actions should not be an empty array."
        if device_mem and teacher is None and not (trace or keep_tree or stepwise or continue_tree):
            return self._search_device(n, obs, legal_mask, to_play, add_exploration_noise, noise, first_index, game_id,
                                       move_index)
        io = _lib.MzSearchIO()
        io.n_games = n
        io.mem = _lib.MZ_MEM_DEVICE if device_mem else _lib.MZ_MEM_HOST
        if obs is not None:
            if not device_mem:
                obs = numpy.asarray(obs, dtype=numpy.float32).reshape(n, -1)
                if obs.shape[1] != self.obs_elems:
                    raise ValueError(f"observation has {obs.shape[1]} elements, expected {self.obs_elems}")
            io.obs = self._ptr(obs, numpy.float32, keep)
        io.legal_mask = self._ptr(legal_mask, numpy.uint8, keep)
        io.to_play = self._ptr(to_play, numpy.int32, keep)
        io.add_exploration_noise = int(bool(add_exploration_noise))
        io.flags = ((_lib.MZ_FLAG_KEEP_TREE if keep_tree else 0) | (_lib.MZ_FLAG_STEPWISE if stepwise else 0)
                    | (_lib.MZ_FLAG_CONTINUE if continue_tree else 0))
        io.noise = self._ptr(noise, numpy.float64, keep)
        io.first_index = self._ptr(first_index, numpy.int32, keep)
        io.game_id = self._ptr(game_id, numpy.int64, keep)
        io.move_index = self._ptr(move_index, numpy.int32, keep)

        if device_mem:
            import torch
            dev = obs.device
            mk = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
            out = SearchOutput(mk((n, A), torch.int32), mk((n,), torch.float64), mk((n,), torch.float32),
                               mk((n,), torch.int32), mk((n,), torch.int32), mk((n, A), torch.float64),
                               mk((n, 2), torch.float64))
            p = lambda t: t.data_ptr()
        else:
            out = SearchOutput(numpy.empty((n, A), numpy.int32), numpy.empty(n, numpy.float64),
                               numpy.empty(n, numpy.float32), numpy.empty(n, numpy.int32), numpy.empty(n, numpy.int32),
                               numpy.empty((n, A), numpy.float64), numpy.empty((n, 2), numpy.float64))
            p = lambda a: a.ctypes.data
        io.visit_counts, io.root_value, io.root_predicted_value = p(out.visit_counts), p(out.root_value), p(out.root_predicted_value)
        io.max_tree_depth, io.tie_count, io.root_priors = p(out.max_tree_depth), p(out.tie_count), p(out.root_priors)
        io.value_range = p(out.value_range)

        if teacher is not None:
            t = _lib.MzTeacher()
            for f in ("root_value", "root_reward", "root_priors", "value", "reward", "priors"):
                setattr(t, f, self._ptr(teacher[f], numpy.float32, keep))
            keep.append(t)
            io.teacher = C.pointer(t)
        if trace:
            if device_mem:
                raise ValueError("trace is only available with host buffers")
            D = int(trace_depth or max(1, N))
            tr = dict(depth=numpy.zeros((n, N), numpy.int32), actions=numpy.zeros((n, N, D), numpy.uint8),
                      value=numpy.zeros((n, N), numpy.float32), reward=numpy.zeros((n, N), numpy.float32),
                      priors=numpy.zeros((n, N, A), numpy.float32), root_priors_raw=numpy.zeros((n, A), numpy.float32),
                      root_reward=numpy.zeros(n, numpy.float32), noise=numpy.zeros((n, A), numpy.float64))
            t = _lib.MzTrace()
            t.max_depth = D
            for k, v in tr.items():
                setattr(t, k, v.ctypes.data)
            keep.append(t)
            io.trace = C.pointer(t)
            out.trace = tr
        self._check(self.lib.mz_search(self._h, C.byref(io)))
        out.device_ms = self.last_search_ms
        return out

    def _search_device(self, n, obs, legal_mask, to_play, add_noise, noise, first_index, game_id, move_index):
        """search() on device tensors through mz_search_device: the seven outputs are views of one buffer, carved while
        the search runs.  The buffer of the next search of as many games on the same device is allocated while this one
        runs too; every buffer belongs to one search only, so returned arrays stay valid as long as the caller holds them."""
        import torch
        keep, io = [], self._dio
        io.n_games = n
        io.add_exploration_noise = 1 if add_noise else 0
        io.obs = self._ptr(obs, numpy.float32, keep)
        io.noise = self._ptr(noise, numpy.float64, keep)
        io.game_id = self._ptr(game_id, numpy.int64, keep)
        io.move_index = self._ptr(move_index, numpy.int32, keep)
        io.legal_mask = self._ptr(legal_mask, numpy.uint8, keep)
        io.to_play = self._ptr(to_play, numpy.int32, keep)
        io.first_index = self._ptr(first_index, numpy.int32, keep)
        key = (n, obs.get_device())
        nxt, self._next_out = self._next_out, None
        if nxt is not None and nxt[0] == key:
            buf, fields, offsets = nxt[1]
        else:
            fields, nbytes = output_layout(n, self.A)
            offsets = tuple(f[3] for f in fields)
            buf = torch.empty(nbytes // 8, dtype=torch.float64, device=obs.device)
        base = buf.data_ptr()
        (io.visit_counts, io.root_value, io.root_predicted_value, io.max_tree_depth, io.tie_count, io.root_priors,
         io.value_range) = (base + o for o in offsets)
        self._check(self.lib.mz_search_device(self._h, self._dio_ref))
        try:
            out = carve_outputs(buf, fields)
            self._next_out = (key, (torch.empty_like(buf), fields, offsets))
        finally:
            self._check(self.lib.mz_search_device_wait(self._h, self._dio_ref))
        out.device_ms = io.device_ms
        return out

    # ------------------------------------------------------------------ networks
    def _inference(self, fn, n, x, action):
        A, F, H = self.A, self.spec.full_support, self.hidden_elems
        keep = []
        res = dict(value_logits=numpy.empty((n, F), numpy.float32), reward_logits=numpy.empty((n, F), numpy.float32),
                   policy_logits=numpy.empty((n, A), numpy.float32), hidden=numpy.empty((n, H), numpy.float32),
                   value=numpy.empty(n, numpy.float32), reward=numpy.empty(n, numpy.float32))
        o = _lib.MzInferenceOut()
        for k, v in res.items():
            setattr(o, k, v.ctypes.data)
        xp = self._ptr(numpy.asarray(x, dtype=numpy.float32).reshape(n, -1), numpy.float32, keep)
        if action is None:
            self._check(fn(self._h, n, _lib.MZ_MEM_HOST, xp, C.byref(o)))
        else:
            ap = self._ptr(numpy.asarray(action).reshape(n), numpy.int32, keep)
            self._check(fn(self._h, n, _lib.MZ_MEM_HOST, xp, ap, C.byref(o)))
        return res

    def initial_inference(self, obs):
        obs = numpy.asarray(obs, dtype=numpy.float32)
        return self._inference(self.lib.mz_initial_inference, obs.shape[0], obs, None)

    def recurrent_inference(self, hidden, action):
        hidden = numpy.asarray(hidden, dtype=numpy.float32)
        return self._inference(self.lib.mz_recurrent_inference, hidden.shape[0], hidden, action)

    # ------------------------------------------------------------------ Reanalyse
    def _reanalyse_io(self, frames, frame_offsets, actions, action_offsets, positions, stacked_observations, keep):
        """MzReanalyseIO over numpy arrays (host) or CUDA torch tensors (device) of frames [F][O] and actions."""
        device_mem = _is_torch(frames)
        if not device_mem:
            frames = numpy.asarray(frames, dtype=numpy.float32)
        O = int(frames.shape[1]) if frames.ndim == 2 else int(numpy.prod(tuple(frames.shape[1:]), dtype=numpy.int64))
        io = _lib.MzReanalyseIO()
        positions = numpy.ascontiguousarray(positions, dtype=numpy.int64)
        io.n_games = len(positions)
        io.mem = _lib.MZ_MEM_DEVICE if device_mem else _lib.MZ_MEM_HOST
        io.stacked_observations = int(self.config.stacked_observations if stacked_observations is None
                                      else stacked_observations)
        io.frame_elems = O
        io.frames = self._ptr(frames, numpy.float32, keep)
        io.actions = self._ptr(actions, numpy.int32, keep)
        io.frame_offsets = self._ptr(numpy.asarray(frame_offsets, dtype=numpy.int64), numpy.int64, keep)
        io.action_offsets = self._ptr(numpy.asarray(action_offsets, dtype=numpy.int64), numpy.int64, keep)
        io.positions = self._ptr(positions, numpy.int64, keep)
        return io, int(positions.sum()), device_mem

    def reanalyse_values(self, frames, frame_offsets, actions, action_offsets, positions, stacked_observations=None):
        """Fresh root values of every position of a batch of games (mz_reanalyse_values): game g's frames are rows
        [frame_offsets[g], frame_offsets[g + 1]) of ``frames`` ([F][O] float32), its action history (leading 0
        included) entries [action_offsets[g], action_offsets[g + 1]) of ``actions``, its positions 0 .. positions[g] - 1.
        Returns float32 [sum positions] in game order: a numpy array for host frames, a CUDA tensor for CUDA frames and
        actions."""
        keep = []
        io, total, device_mem = self._reanalyse_io(frames, frame_offsets, actions, action_offsets, positions,
                                                   stacked_observations, keep)
        if device_mem:
            import torch
            values = torch.empty(total, dtype=torch.float32, device=frames.device)
            io.values = values.data_ptr() if total else None
        else:
            values = numpy.empty(total, numpy.float32)
            io.values = values.ctypes.data if total else None
        self._check(self.lib.mz_reanalyse_values(self._h, C.byref(io)))
        return values

    def reanalyse_search(self, frames, frame_offsets, actions, action_offsets, positions, legal_mask=None, to_play=None,
                         game_id=None, add_exploration_noise=True, stacked_observations=None):
        """The self-play search re-run at every position of a batch of games (mz_reanalyse_search): the positions are
        reanalyse_values', ``legal_mask`` [sum positions][A] and ``to_play`` [sum positions] are theirs in game order,
        ``game_id`` [n games] keys each game's Philox streams (the move index is the position).  Returns
        (visit_counts int32 [sum positions][A], root_value float64 [sum positions]): numpy arrays for host frames, CUDA
        tensors for CUDA frames, actions, legal masks and to_play."""
        keep = []
        io, total, device_mem = self._reanalyse_io(frames, frame_offsets, actions, action_offsets, positions,
                                                   stacked_observations, keep)
        if device_mem:
            import torch
            to_dev = lambda x, dt: x if x is None or _is_torch(x) else torch.as_tensor(numpy.asarray(x, dt), device=frames.device)
            legal_mask, to_play = to_dev(legal_mask, numpy.uint8), to_dev(to_play, numpy.int32)
        sio = _lib.MzReanalyseSearchIO()
        sio.games = C.addressof(io)
        sio.legal_mask = self._ptr(legal_mask, numpy.uint8, keep)
        sio.to_play = self._ptr(to_play, numpy.int32, keep)
        sio.game_id = self._ptr(None if game_id is None else numpy.asarray(game_id, dtype=numpy.int64).reshape(-1),
                                numpy.int64, keep)
        sio.add_exploration_noise = int(bool(add_exploration_noise))
        if device_mem:
            visits = torch.empty((total, self.A), dtype=torch.int32, device=frames.device)
            root = torch.empty(total, dtype=torch.float64, device=frames.device)
            p = lambda t: t.data_ptr() if total else None
        else:
            visits = numpy.empty((total, self.A), numpy.int32)
            root = numpy.empty(total, numpy.float64)
            p = lambda a: a.ctypes.data if total else None
        sio.visit_counts, sio.root_value = p(visits), p(root)
        self._check(self.lib.mz_reanalyse_search(self._h, C.byref(sio)))
        return visits, root

    def debug_reanalyse_stack(self, chunk, frames, frame_offsets, actions, action_offsets, positions,
                              stacked_observations=None):
        """The stacked inputs [n_c][obs_elems] chunk ``chunk`` of reanalyse_values builds (mz_debug_reanalyse_stack)."""
        keep = []
        io, total, _ = self._reanalyse_io(frames, frame_offsets, actions, action_offsets, positions, stacked_observations,
                                          keep)
        n = max(0, min(self.max_games, total - int(chunk) * self.max_games))
        out = numpy.empty((n, self.obs_elems), numpy.float32)
        self._check(self.lib.mz_debug_reanalyse_stack(self._h, C.byref(io), int(chunk), out.ctypes.data if n else None))
        return out

    # ------------------------------------------------------------------ tree
    def export_tree(self, game: int, with_hidden: bool = False):
        S = (self.pool_n + 1) * self.A
        out = dict(child_visit=numpy.zeros(S, numpy.int32), child_value_sum=numpy.zeros(S, numpy.float64),
                   child_reward=numpy.zeros(S, numpy.float32), child_prior=numpy.zeros(S, numpy.float64),
                   child_expansion=numpy.full(S, -1, numpy.int32))
        e = _lib.MzTreeExport()
        for k, v in out.items():
            setattr(e, k, v.ctypes.data)
        if with_hidden:
            out["hidden"] = numpy.zeros((self.pool_n + 1, self.hidden_elems), numpy.float32)
            e.hidden = out["hidden"].ctypes.data
        self._check(self.lib.mz_export_tree(self._h, int(game), C.byref(e)))
        out["n_expansions"] = int(e.n_expansions)
        out["root_visit"] = int(e.root_visit)
        out["root_value_sum"] = float(e.root_value_sum)
        out["root_reward"] = float(e.root_reward)
        return out

    def import_tree(self, game: int, tree: dict):
        """Seed game ``game``'s tree in the node pool (the inverse of ``export_tree``; ``mz_import_tree``): arrays
        ``child_visit / child_value_sum / child_reward / child_prior / child_expansion`` of ``n_expansions * A`` entries,
        ``hidden [n_expansions, hidden_elems]``, ``root_visit``, ``root_value_sum``, ``root_reward``."""
        keep = []
        K = int(tree["n_expansions"])
        e = _lib.MzTreeExport()
        e.n_expansions = K
        for k, dt in (("child_visit", numpy.int32), ("child_value_sum", numpy.float64), ("child_reward", numpy.float32),
                      ("child_prior", numpy.float64), ("child_expansion", numpy.int32)):
            a = numpy.ascontiguousarray(tree[k], dtype=dt).reshape(-1)
            assert a.size >= K * self.A, k
            keep.append(a)
            setattr(e, k, a.ctypes.data)
        if tree.get("hidden") is not None:
            hdn = numpy.ascontiguousarray(tree["hidden"], dtype=numpy.float32).reshape(-1)
            assert hdn.size >= K * self.hidden_elems
            keep.append(hdn)
            e.hidden = hdn.ctypes.data
        e.root_visit = int(tree["root_visit"])
        e.root_value_sum = float(tree["root_value_sum"])
        e.root_reward = float(tree.get("root_reward", 0.0))
        self._check(self.lib.mz_import_tree(self._h, int(game), C.byref(e)))


class DeviceSelfPlayLoop:
    """Python face of mz_selfplay_*: ``max_games`` environments stepped on the GPU, one batched search per move,
    finished games handed back as packed struct-of-arrays blocks (SURVEY.md 8f-1, include/mzb200.h)."""

    ENVS = {"cartpole": _lib.MZ_ENV_CARTPOLE, "tictactoe": _lib.MZ_ENV_TICTACTOE, "connect4": _lib.MZ_ENV_CONNECT4,
            "gomoku": _lib.MZ_ENV_GOMOKU, "twentyone": _lib.MZ_ENV_TWENTYONE, "simple_grid": _lib.MZ_ENV_SIMPLE_GRID,
            "gridworld": _lib.MZ_ENV_GRIDWORLD}
    OPPONENTS = {"self": _lib.MZ_OPPONENT_SELF, "expert": _lib.MZ_OPPONENT_EXPERT, "random": _lib.MZ_OPPONENT_RANDOM}

    def __init__(self, engine: SearchEngine, env: str, max_moves: int, temperature_threshold=None, reward_scale: int = 1,
                 first_game_id: int = 0, staging_bytes: int = 0, game_id_stride: int = 0, td_steps: int = 0,
                 per_alpha: float = 1.0, discount: float = 1.0, opponent: str = "self", muzero_player: int = 0,
                 stacked_observations: int = 0):
        """``opponent`` "expert" or "random" plays test-mode games (``play_game(..., opponent, muzero_player)``): the
        opponent's moves are played on the device and recorded with a NaN root value and zero visit counts.  An opponent
        the game lacks (Gomoku's "expert") raises NotImplementedError.  ``stacked_observations`` (the config's; the
        engine's network must have been built for it) makes every search see the stacked input of
        ``get_stacked_observations``, built on the device; the staged observations stay the environment's own."""
        if env not in self.ENVS:
            raise NotImplementedError(f"no device-resident environment for {env!r}")
        if opponent not in self.OPPONENTS:
            raise NotImplementedError(f"no device opponent {opponent!r} (expected one of {sorted(self.OPPONENTS)})")
        self.engine = engine
        self.opponent, self.muzero_player = opponent, int(muzero_player)
        d = self._desc(self.ENVS[env], max_moves, temperature_threshold, reward_scale, first_game_id, staging_bytes,
                       game_id_stride, td_steps, per_alpha, discount, stacked_observations)
        try:
            engine._check(engine.lib.mz_selfplay_begin_vs(engine._h, C.byref(d), self.OPPONENTS[opponent], self.muzero_player))
        except _lib.MzError as e:
            if e.code == _lib.MZ_EUNSUPPORTED:
                raise NotImplementedError(str(e)) from e
            raise
        self.stats = _lib.MzSelfPlayStats()

    def _desc(self, env, max_moves, temperature_threshold, reward_scale, first_game_id, staging_bytes, game_id_stride,
              td_steps, per_alpha, discount, stacked_observations):
        d = _lib.MzSelfPlayDesc()
        d.env = env
        d.max_moves = int(max_moves)
        d.temperature_threshold = int(temperature_threshold or 0)
        d.reward_scale = int(reward_scale)
        d.first_game_id = int(first_game_id)
        d.game_id_stride = int(game_id_stride)
        d.stacked_observations = int(stacked_observations)
        if td_steps and per_alpha in (0.5, 1, 1.0):
            # PER priorities on the device: discount ** k evaluated HERE, with Python's pow, like replay_buffer.py:246,260
            self._discount_pow = (C.c_double * (int(td_steps) + 1))(*[discount ** k for k in range(int(td_steps) + 1)])
            d.td_steps, d.per_alpha = int(td_steps), float(per_alpha)
            d.discount_pow = C.cast(self._discount_pow, C.c_void_p)
        self.with_priorities = bool(d.td_steps)
        d.staging_bytes = int(staging_bytes)
        return d

    def _inject(self, keep, forced_action, uniform, noise, first_index):
        """MzSelfPlayInject of the given overrides, or None when there are none."""
        if forced_action is None and uniform is None and noise is None and first_index is None:
            return None
        eng = self.engine
        inj = _lib.MzSelfPlayInject()
        inj.forced_action = eng._ptr(forced_action, numpy.int32, keep)
        inj.uniform = eng._ptr(uniform, numpy.float64, keep)
        inj.noise = eng._ptr(noise, numpy.float64, keep)
        inj.first_index = eng._ptr(first_index, numpy.int32, keep)
        return inj

    def moves(self, n_moves: int, temperature: float, forced_action=None, uniform=None, noise=None, first_index=None):
        """Play ``n_moves`` lockstep moves; returns the stats struct (env_steps, games_finished, staged_*, device_ms)."""
        eng = self.engine
        keep = []
        inj = self._inject(keep, forced_action, uniform, noise, first_index)
        eng._check(eng.lib.mz_selfplay_moves(eng._h, int(n_moves), float(temperature),
                                            C.byref(inj) if inj is not None else None, C.byref(self.stats)))
        return self.stats

    def enqueue(self, n_moves: int, temperature: float):
        """Start ``n_moves`` moves without waiting (``mz_selfplay_enqueue``); pair with ``wait``."""
        eng = self.engine
        eng._check(eng.lib.mz_selfplay_enqueue(eng._h, int(n_moves), float(temperature)))

    def wait(self):
        eng = self.engine
        eng._check(eng.lib.mz_selfplay_wait(eng._h, C.byref(self.stats)))
        return self.stats

    def drain_pointers(self):
        """(data address, bytes, games, index address) of the staged games, zero-copy.  The library swaps its two staging
        areas here, so the memory stays intact while the next moves run; copy it before the drain after that."""
        eng = self.engine
        ptr, nbytes, ngames, iptr = C.c_void_p(), C.c_uint64(), C.c_int32(), C.c_void_p()
        eng._check(eng.lib.mz_selfplay_drain(eng._h, C.byref(ptr), C.byref(nbytes), C.byref(ngames), C.byref(iptr)))
        return ptr.value, int(nbytes.value), int(ngames.value), iptr.value

    @staticmethod
    def copy_staged(pointers):
        """``drain_pointers()`` -> (bytes, index[n, 2] uint64) copies."""
        ptr, nbytes, n, iptr = pointers
        if n == 0:
            return b"", numpy.zeros((0, 2), numpy.uint64)
        index = numpy.frombuffer(C.string_at(iptr, 16 * n), numpy.uint64).reshape(n, 2)
        return C.string_at(ptr, nbytes), index

    def drain(self):
        """(bytes, index) of the staged finished games - copies.
        ``index`` is an ``[n, 2]`` uint64 array: byte offset of each game's block, ``(slot << 32) | length``."""
        return self.copy_staged(self.drain_pointers())

    def peek(self):
        eng = self.engine
        B, A = eng.max_games, eng.A
        out = dict(obs=numpy.empty((B, eng.obs_elems), numpy.float32), legal_mask=numpy.empty((B, A), numpy.uint8),
                   to_play=numpy.empty(B, numpy.int32), game_id=numpy.empty(B, numpy.int64),
                   move_index=numpy.empty(B, numpy.int32), last_action=numpy.empty(B, numpy.int32))
        pk = _lib.MzSelfPlayPeek()
        for k, v in out.items():
            setattr(pk, k, v.ctypes.data)
        eng._check(eng.lib.mz_selfplay_peek(eng._h, C.byref(pk)))
        return out


class HostEnvSelfPlayLoop(DeviceSelfPlayLoop):
    """Python face of mz_selfplay_begin_host / _host_act / _host_observe / _host_restart: the device loop for a game
    whose environment the caller steps.  Each move is ``act`` -> [step the environments of the slots whose action is
    >= 0] -> ``observe`` -> [reset the environments of the slots it reports finished] -> ``restart``; ``drain`` and
    ``peek`` are the device loop's.  Rows are ``[max_games, ...]`` arrays (or sequences of per-game arrays)."""

    OBS_HISTORIES = ("device", "host")

    def __init__(self, engine: SearchEngine, obs_shape, max_moves: int, obs, legal_mask, to_play,
                 temperature_threshold=None, first_game_id: int = 0, staging_bytes: int = 0, game_id_stride: int = 0,
                 td_steps: int = 0, per_alpha: float = 1.0, discount: float = 1.0, stacked_observations: int = 0,
                 obs_history: str = "device", opponent: str = "self", muzero_player: int = 0):
        """``obs_shape`` is the environment's (C, H, W); ``obs``, ``legal_mask`` and ``to_play`` the first rows of the
        games ``first_game_id + g``.  ``obs_history`` says who keeps each game's observations: "device" (the staged
        blocks carry them, mz_selfplay_begin_host) or "host" (the device keeps the last stacked_observations + 1 per
        slot, mz_selfplay_begin_host_window, and this object keeps a float32 copy of every row it passes on for the
        game in flight; ``drain`` hands them over with the blocks).  ``opponent`` "expert" or "random" plays test-mode
        games (mz_selfplay_begin_host_vs): after begin, ``observe`` and ``restart``, run the opponent phase
        (``opponent_turn`` / ``opponent_act`` / [step] / ``observe``) until ``opponent_turn`` returns None."""
        if obs_history not in self.OBS_HISTORIES:
            raise ValueError(f"obs_history must be one of {self.OBS_HISTORIES}, got {obs_history!r}")
        if opponent not in self.OPPONENTS:
            raise NotImplementedError(f"no device opponent {opponent!r} (expected one of {sorted(self.OPPONENTS)})")
        self.engine = engine
        self.opponent, self.muzero_player = opponent, int(muzero_player)
        B = engine.max_games
        self.O = int(numpy.prod(obs_shape))
        d = self._desc(_lib.MZ_ENV_HOST, max_moves, temperature_threshold, 0, first_game_id, staging_bytes, game_id_stride,
                       td_steps, per_alpha, discount, stacked_observations)
        e = _lib.MzHostEnvDesc(*(int(x) for x in obs_shape))
        o, lg, tp = self._rows(obs, legal_mask, to_play)
        if opponent == "self" and self.muzero_player == 0:
            begin = engine.lib.mz_selfplay_begin_host if obs_history == "device" else engine.lib.mz_selfplay_begin_host_window
            engine._check(begin(engine._h, C.byref(d), C.byref(e), o.ctypes.data, lg.ctypes.data, tp.ctypes.data))
        else:
            rc = engine.lib.mz_selfplay_begin_host_vs(engine._h, C.byref(d), C.byref(e), self.OPPONENTS[opponent],
                                                      self.muzero_player, int(obs_history == "host"), o.ctypes.data,
                                                      lg.ctypes.data, tp.ctypes.data)
            if rc == _lib.MZ_EUNSUPPORTED:
                raise NotImplementedError(engine.lib.mz_last_error(engine._h).decode())
            engine._check(rc)
        self.obs_history = obs_history
        self.stats = _lib.MzSelfPlayStats()
        self.actions = numpy.empty(B, numpy.int32)
        self.finished = numpy.empty(B, numpy.uint8)
        self.defaults = numpy.empty(B, numpy.int32)
        if obs_history == "host":
            # per slot: its game's id (the library's: first + g, then + stride per restart) and rows so far; the rows of
            # games observe reported finished wait here, by game id, for the drain that returns their blocks
            self._game_id = [int(first_game_id) + g for g in range(B)]
            self._stride = int(game_id_stride) if int(game_id_stride) > 0 else B
            self._rows_of = [[o[g].copy()] for g in range(B)]
            self._finished_rows = {}

    def _rows(self, obs, legal_mask, to_play):
        B = self.engine.max_games
        if not isinstance(obs, numpy.ndarray):
            obs = numpy.stack([numpy.asarray(x) for x in obs])
        return (numpy.ascontiguousarray(obs, numpy.float32).reshape(B, self.O),
                numpy.ascontiguousarray(legal_mask, numpy.uint8).reshape(B, self.engine.A),
                numpy.ascontiguousarray(to_play, numpy.int32).reshape(B))

    def act(self, temperature: float, forced_action=None, uniform=None, noise=None, first_index=None):
        """One batched search and the action of every slot: an int32 ``[max_games]`` array (reused by the next call),
        -1 for a slot that is not playing this move (its finished game waits for staging space)."""
        eng = self.engine
        keep = []
        inj = self._inject(keep, forced_action, uniform, noise, first_index)
        eng._check(eng.lib.mz_selfplay_host_act(eng._h, float(temperature), C.byref(inj) if inj is not None else None,
                                               self.actions.ctypes.data))
        return self.actions

    def opponent_turn(self):
        """The random default of every slot whose opponent move is due, -1 for the others: an int32 ``[max_games]``
        array (reused by the next call), or None when no opponent move is due and MuZero moves next."""
        eng = self.engine
        n = eng.lib.mz_selfplay_host_opponent_turn(eng._h, self.defaults.ctypes.data)
        eng._check(min(n, 0))
        return self.defaults if n > 0 else None

    def opponent_act(self, actions=None):
        """The opponent's moves of the slots ``opponent_turn`` found: ``actions`` (an int array ``[max_games]``, read at
        those slots) or, when None, their random defaults.  Returns the moves as ``act`` does, -1 for the slots without
        one: step those with a move, then ``observe``."""
        eng = self.engine
        a = None if actions is None else numpy.ascontiguousarray(actions, numpy.int32).reshape(-1)
        eng._check(eng.lib.mz_selfplay_host_opponent_act(eng._h, None if a is None else a.ctypes.data,
                                                        self.actions.ctypes.data))
        return self.actions

    def observe(self, obs, reward, done, legal_mask, to_play):
        """The step's rows for the whole batch (rows of slots that did not play are ignored); ``reward`` is rounded once to
        float32.  Returns the bool ``[max_games]`` mask of the slots whose game ended and was packed (reset them, then
        ``restart``); the stats struct is ``self.stats``."""
        eng = self.engine
        o, lg, tp = self._rows(obs, legal_mask, to_play)
        r = numpy.ascontiguousarray(numpy.asarray(reward, numpy.float64).astype(numpy.float32).reshape(-1))
        dn = numpy.ascontiguousarray(numpy.asarray(done).astype(numpy.uint8).reshape(-1))
        eng._check(eng.lib.mz_selfplay_host_observe(eng._h, o.ctypes.data, r.ctypes.data, dn.ctypes.data, lg.ctypes.data,
                                                   tp.ctypes.data, self.finished.ctypes.data, C.byref(self.stats)))
        finished = self.finished.astype(bool)
        if self.obs_history == "host":
            for g in numpy.nonzero(self.actions >= 0)[0]:        # a parked slot's row is not its game's
                self._rows_of[g].append(o[g].copy())
            for g in numpy.nonzero(finished)[0]:
                self._finished_rows[self._game_id[g]] = numpy.stack(self._rows_of[g])
                self._rows_of[g] = None
        return finished

    def restart(self, which, obs, legal_mask, to_play):
        """The first rows of the next games of the slots of ``which`` (the mask ``observe`` returned, or part of it)."""
        eng = self.engine
        w = numpy.ascontiguousarray(numpy.asarray(which).astype(numpy.uint8).reshape(-1))
        o, lg, tp = self._rows(obs, legal_mask, to_play)
        eng._check(eng.lib.mz_selfplay_host_restart(eng._h, w.ctypes.data, o.ctypes.data, lg.ctypes.data, tp.ctypes.data))
        if self.obs_history == "host":
            for g in numpy.nonzero(w)[0]:
                self._game_id[g] += self._stride
                self._rows_of[g] = [o[g].copy()]

    def drain(self):
        """(bytes, index) of the staged finished games, as ``DeviceSelfPlayLoop.drain``; with ``obs_history="host"``
        also ``{game id: [T + 1, O] float32}``, the observations of those games (their blocks carry none)."""
        buf, index = super().drain()
        if self.obs_history == "device":
            return buf, index
        ids = [int(numpy.frombuffer(buf, numpy.int64, 1, int(off))[0]) for off in index[:, 0]]
        return buf, index, {gid: self._finished_rows.pop(gid) for gid in ids}


class UserEnvSelfPlayLoop(DeviceSelfPlayLoop):
    """Python face of mz_selfplay_begin_user / _user_moves: the device loop for a game whose environment is CUDA source
    (``source`` defines ``mz_env_reset`` and ``mz_env_step`` against csrc/user_env.cuh; ``state_bytes`` per slot).  The
    library compiles the source with NVRTC for sm_90a, once per handle and source.  ``moves``, ``enqueue`` / ``wait``,
    ``drain`` and ``peek`` are the device loop's.

    ``opponent`` "expert" or "random" plays test-mode games (mz_selfplay_begin_user_vs): every move is MuZero's pass,
    then two passes of the opponent's moves, stepped by the same source; "expert" needs a source that defines
    ``MZ_ENV_EXPERT`` and ``mz_env_expert`` (csrc/user_env_expert.cuh), else NotImplementedError."""

    def __init__(self, engine: SearchEngine, source: str, state_bytes: int, obs_shape, max_moves: int,
                 temperature_threshold=None, first_game_id: int = 0, staging_bytes: int = 0, game_id_stride: int = 0,
                 td_steps: int = 0, per_alpha: float = 1.0, discount: float = 1.0, stacked_observations: int = 0,
                 opponent: str = "self", muzero_player: int = 0):
        if opponent not in self.OPPONENTS:
            raise NotImplementedError(f"no device opponent {opponent!r} (expected one of {sorted(self.OPPONENTS)})")
        self.engine = engine
        self.opponent, self.muzero_player = opponent, int(muzero_player)
        d = self._desc(_lib.MZ_ENV_USER, max_moves, temperature_threshold, 0, first_game_id, staging_bytes, game_id_stride,
                       td_steps, per_alpha, discount, stacked_observations)
        self._source = source.encode()
        e = _lib.MzUserEnvDesc(self._source, int(state_bytes), *(int(x) for x in obs_shape))
        if opponent == "self" and self.muzero_player == 0:
            rc = engine.lib.mz_selfplay_begin_user(engine._h, C.byref(d), C.byref(e))
        else:
            rc = engine.lib.mz_selfplay_begin_user_vs(engine._h, C.byref(d), C.byref(e), self.OPPONENTS[opponent],
                                                      self.muzero_player)
        if rc == _lib.MZ_EUNSUPPORTED:
            raise NotImplementedError(engine.lib.mz_last_error(engine._h).decode())
        engine._check(rc)
        self.stats = _lib.MzSelfPlayStats()

    def moves(self, n_moves: int, temperature: float, forced_action=None, uniform=None, noise=None, first_index=None):
        eng = self.engine
        keep = []
        inj = self._inject(keep, forced_action, uniform, noise, first_index)
        eng._check(eng.lib.mz_selfplay_user_moves(eng._h, int(n_moves), float(temperature),
                                                 C.byref(inj) if inj is not None else None, C.byref(self.stats)))
        return self.stats

    @property
    def compiles(self):
        """NVRTC compiles made for this engine's user environments so far."""
        return int(self.engine.lib.mz_debug_user_env_compiles(self.engine._h))


def debug_user_env_compile(source: str, log_bytes: int = 1 << 16):
    """Compiles a user environment's source as mz_selfplay_begin_user does, on the host (no GPU needed).  Returns
    ``(rc, log, info)``: the library's return code, NVRTC's log (ptxas's resource report included) and a dict of the
    wrapper kernels' ``{kernel: (registers, stack frame bytes, spill store bytes, spill load bytes)}`` plus
    ``"nvrtc_version"``; ``mz_last_error(NULL)`` holds the reason of a failure."""
    lib = _lib.load_library()
    log = C.create_string_buffer(int(log_bytes))
    info = (C.c_int32 * 9)()
    rc = lib.mz_debug_user_env_compile(source.encode(), log, int(log_bytes), info)
    return rc, log.value.decode(), {"reset": tuple(info[0:4]), "step": tuple(info[4:8]), "nvrtc_version": int(info[8])}


def debug_user_env_expert_compile(source: str, log_bytes: int = 1 << 16):
    """``debug_user_env_compile`` with the expert wrapper (mz_debug_user_env_expert_compile): the info dict has
    ``"expert"`` (True when the source defines MZ_ENV_EXPERT and the wrapper was compiled) and ``"expert_kernel"``, its
    (registers, stack frame bytes, spill store bytes, spill load bytes), -1s without one."""
    lib = _lib.load_library()
    log = C.create_string_buffer(int(log_bytes))
    info = (C.c_int32 * 14)()
    rc = lib.mz_debug_user_env_expert_compile(source.encode(), log, int(log_bytes), info)
    return rc, log.value.decode(), {"reset": tuple(info[0:4]), "step": tuple(info[4:8]), "nvrtc_version": int(info[8]),
                                    "expert": bool(info[9]), "expert_kernel": tuple(info[10:14])}


def parse_staged_game(buf: bytes, off: int):
    """One packed block of ``mz_selfplay_drain`` -> dict of numpy views into ``buf`` (no copies)."""
    H = _lib.MZ_STAGED_HEADER_BYTES
    gid = int(numpy.frombuffer(buf, numpy.int64, 1, off)[0])
    slot, T, first_to_play, O, A, nbytes = (int(x) for x in numpy.frombuffer(buf, numpy.int32, 6, off + 8))
    p = off + H
    root = numpy.frombuffer(buf, numpy.float64, T, p); p += 8 * T
    visits = numpy.frombuffer(buf, numpy.int32, T * A, p).reshape(T, A); p += 4 * T * A
    action = numpy.frombuffer(buf, numpy.int32, T, p); p += 4 * T
    reward = numpy.frombuffer(buf, numpy.float32, T, p); p += 4 * T
    to_play = numpy.frombuffer(buf, numpy.int32, T, p); p += 4 * T
    priority = numpy.frombuffer(buf, numpy.float32, T, p); p += 4 * T
    obs = numpy.frombuffer(buf, numpy.float32, (T + 1) * O, p).reshape(T + 1, O)
    return dict(game_id=gid, slot=slot, length=T, first_to_play=first_to_play, root_value=root, visits=visits,
                action=action, reward=reward, to_play=to_play, priority=priority, obs=obs, bytes=nbytes)


def parse_staged_games(buf: bytes, index):
    """All staged games of one drain, in staging order."""
    games = [parse_staged_game(buf, int(off)) for off in index[:, 0]]
    assert sum(g["bytes"] for g in games) == len(buf), "staged blocks do not add up"
    for g, meta in zip(games, index[:, 1]):
        assert (int(meta) >> 32, int(meta) & 0xFFFFFFFF) == (g["slot"], g["length"])
    return games


def debug_opponent_action(env, boards, players, uniforms=None, defaults=None, opponent="expert", device=0):
    """The device opponent of test-mode games on host positions (mz_debug_opponent_action).  ``boards`` is
    ``[n, H, W]`` (or ``[n, H*W]``) of +1 / -1 / 0 with row 0 at the bottom, ``players`` ``[n]`` the side to move
    (+1 / -1).  The random default is the legal action with index ``floor(u * n_legal)`` for ``uniforms[i]``, or
    ``defaults[i]`` when given.  Returns the ``[n]`` int32 actions."""
    lib = _lib.load_library()
    codes = {"tictactoe": _lib.MZ_ENV_TICTACTOE, "connect4": _lib.MZ_ENV_CONNECT4, "gomoku": _lib.MZ_ENV_GOMOKU}
    if env not in codes:
        raise NotImplementedError(f"no device opponent for {env!r}")
    b = numpy.ascontiguousarray(boards, numpy.int8)
    n = b.shape[0]
    b = b.reshape(n, -1)
    p = numpy.ascontiguousarray(players, numpy.int8).reshape(n)
    u = None if uniforms is None else numpy.ascontiguousarray(uniforms, numpy.float64).reshape(n)
    d = None if defaults is None else numpy.ascontiguousarray(defaults, numpy.int32).reshape(n)
    out = numpy.empty(n, numpy.int32)
    rc = lib.mz_debug_opponent_action(device, codes[env], DeviceSelfPlayLoop.OPPONENTS[opponent], n, b.ctypes.data,
                                      p.ctypes.data, None if u is None else u.ctypes.data,
                                      None if d is None else d.ctypes.data, out.ctypes.data)
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    return out


def debug_conv3x3(x, w, bias=None, residual=None, relu=False, tensor_cores=False, device=0, stride=1):
    """One conv3x3 (pad 1, stride 1 or 2) on the device through mz_debug_conv3x3; numpy NCHW in and out.
    x is [n, Cin, H, W], w [Cout, Cin, 3, 3], bias [Cout], residual and the result [n, Cout, Ho, Wo].
    ``tensor_cores``: False / "off" = CUDA cores, "fp16" = wgmma with fp16 operands, True / "x3" = wgmma on split operands."""
    lib = _lib.load_library()
    x = numpy.ascontiguousarray(x, numpy.float32)
    w = numpy.ascontiguousarray(w, numpy.float32)
    n, cin, H, W = x.shape
    cout = w.shape[0]
    if w.shape != (cout, cin, 3, 3):
        raise ValueError(f"weights {w.shape} do not fit {cin} input channels")
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = numpy.empty((n, cout, Ho, Wo), numpy.float32)
    b = None if bias is None else numpy.ascontiguousarray(bias, numpy.float32)
    r = None if residual is None else numpy.ascontiguousarray(residual, numpy.float32)
    if b is not None and b.shape != (cout,):
        raise ValueError(f"bias {b.shape} does not fit {cout} output channels")
    if r is not None and r.shape != out.shape:
        raise ValueError(f"residual {r.shape} does not match the output {out.shape}")
    mode = {False: 0, True: 2, "off": 0, "fp16": 1, "x3": 2}[tensor_cores]
    rc = lib.mz_debug_conv3x3(device, n, cin, cout, H, W, stride, x.ctypes.data, w.ctypes.data,
                              None if b is None else b.ctypes.data, None if r is None else r.ctypes.data, int(relu), mode,
                              out.ctypes.data)
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    return out


TOWER_SITES = {"representation": 0, "dynamics": 1, "dynamics_pool": 2, "prediction": 3}


def _tower_args(x, weights, biases, site, actions, parents, channels=None):
    """Validates one debug tower call and marshals it for the entry: returns (the tower's channels, its blocks, the arrays
    x, weights, biases, actions, parents in the entries' order, None where not given).  ``channels``: 64 or 128 for the
    tensor-core towers, which leave the representation stem to the CUDA cores; None for the fused CUDA-core tower, which
    takes that stem and any channel count (the first conv's outputs)."""
    x = numpy.ascontiguousarray(x, numpy.float32)
    n, cin, H, W = x.shape
    fused = channels is None
    dyn = site in ("dynamics", "dynamics_pool")
    stem = dyn or (fused and site == "representation")
    ch = numpy.shape(weights[0])[0] if fused else channels
    if (len(weights) - stem) % 2 != 0 or (cin != ch and not (stem and not dyn)):
        raise ValueError(f"{cin} input planes / {len(weights)} convs do not make a {ch}-channel tower at site {site}")
    for i, w in enumerate(weights):
        want = (ch, (ch + 1 if dyn else cin) if stem and i == 0 else ch, 3, 3)
        if numpy.shape(w) != want:
            raise ValueError(f"conv {i}: weights {numpy.shape(w)}, expected {want}")
    wcat = numpy.ascontiguousarray(numpy.concatenate([numpy.asarray(w, numpy.float32).reshape(-1) for w in weights]))
    b = None if biases is None else numpy.ascontiguousarray(numpy.stack(biases), numpy.float32)
    if b is not None and b.shape != (len(weights), ch):
        raise ValueError(f"biases {b.shape} do not fit {len(weights)} convs")
    act = None if actions is None else numpy.ascontiguousarray(actions, numpy.int32)
    par = None if parents is None else numpy.ascontiguousarray(parents, numpy.int32)
    return ch, (len(weights) - stem) // 2, (x, wcat, b, act, par)


def _ptrs(arrays):
    return [None if a is None else a.ctypes.data for a in arrays]


def debug_conv_tower(x, weights, biases=None, mode="x3", site="prediction", actions=None, A=1, parents=None,
                     pool_stride=1, parts=1, device=0):
    """One 64-channel tensor-core tower of a network call site through mz_debug_conv_tower; numpy NCHW in and out.
    x is [n, 64, H, W]; ``weights`` the convs in order ([64, 65, 3, 3] dynamics stem first, then two [64, 64, 3, 3] per
    block), ``biases`` one [64] per conv.  ``site``: "representation", "dynamics" (plain recurrent call), "dynamics_pool"
    (in search: game g's input in pool slot ``parents[g]`` of ``pool_stride``; ``parts`` ranges of the partitioned
    replay) or "prediction".  Returns (out [n, 64, H, W], kernel launches, x3 range-guard count)."""
    lib = _lib.load_library()
    _, blocks, arrays = _tower_args(x, weights, biases, site, actions, parents, 64)
    n, _, H, W = arrays[0].shape
    out = numpy.empty_like(arrays[0])
    launches, sat = C.c_int64(0), C.c_int32(0)
    rc = lib.mz_debug_conv_tower(device, n, H, W, {"fp16": 1, "x3": 2}[mode], blocks, TOWER_SITES[site], parts, A,
                                 *_ptrs(arrays), pool_stride, out.ctypes.data, C.byref(launches), C.byref(sat))
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    return out, launches.value, sat.value


SMALL_TOWER_PLAN = ("P", "CO", "boards", "threads", "grid", "smem")


def debug_small_tower_plan(n, in_channels, channels, H, W, blocks, stem, sm_count):
    """Launch plan of the fused CUDA-core tower (mz_debug_small_tower_plan, host only): (a dict of P, CO, boards per CTA,
    threads, grid and smem, "") or (None, the reason) when the fused tower refuses the shape.  ``in_channels``: planes
    the stem reads (C + 1 for the dynamics stem); without a stem, ``channels``."""
    lib = _lib.load_library()
    out = (C.c_int64 * 6)()
    if not lib.mz_debug_small_tower_plan(n, in_channels, channels, H, W, blocks, int(stem), sm_count, out):
        return None, lib.mz_last_error(None).decode()
    return dict(zip(SMALL_TOWER_PLAN, out)), ""

def debug_small_tower(x, weights, biases=None, site="prediction", actions=None, A=1, parents=None, pool_stride=1, parts=1,
                      device=0):
    """One fused CUDA-core tower of a network call site through mz_debug_small_tower; numpy NCHW in and out.  ``weights``
    are the convs in order ([C, cin, 3, 3]: the stem first, cin = x's planes at "representation" and C + 1 at the dynamics
    sites, then two [C, C, 3, 3] per block), ``biases`` one [C] per conv.  ``site``: "representation", "dynamics" (plain
    recurrent call), "dynamics_pool" (in search: game g's input in pool slot ``parents[g]`` of ``pool_stride``; ``parts``
    ranges of the partitioned replay) or "prediction".  Returns (out [n, C, H, W], the plan of the launch as a dict)."""
    lib = _lib.load_library()
    ch, blocks, arrays = _tower_args(x, weights, biases, site, actions, parents)
    n, cin, H, W = arrays[0].shape
    out = numpy.empty((n, ch, H, W), numpy.float32)
    plan = (C.c_int64 * 6)()
    rc = lib.mz_debug_small_tower(device, n, cin, ch, H, W, blocks, TOWER_SITES[site], parts, A, *_ptrs(arrays),
                                  pool_stride, out.ctypes.data, plan)
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    return out, dict(zip(SMALL_TOWER_PLAN, plan))


WIDE_TOWER_PLAN = ("m_tiles", "threads", "smem", "stages", "layers", "ctas_per_sm", "wave", "launches", "reg_cap")


WIDE_PAIR_TOWER_PLAN = ("rows0", "m_tiles", "threads", "smem", "stages", "layers", "wave", "launches", "reg_cap")


def debug_wide_tower_plan(n, channels, H, W, blocks, stem, sm_count):
    """Launch plan of the 128-channel x3 tensor-core tower (mz_debug_wide_tower_plan, host only): (a dict of
    WIDE_TOWER_PLAN, "") or (None, the reason) when the wide towers refuse the shape."""
    return _wide_plan("mz_debug_wide_tower_plan", WIDE_TOWER_PLAN, n, channels, H, W, blocks, stem, sm_count)


def debug_wide_pair_tower_plan(n, channels, H, W, blocks, stem, sm_count):
    """Launch plan of the same tower with each board split across a CTA pair (mz_debug_wide_pair_tower_plan, host only):
    (a dict of WIDE_PAIR_TOWER_PLAN, per-CTA figures except ``wave``, the boards per wave), "") or (None, the reason)."""
    return _wide_plan("mz_debug_wide_pair_tower_plan", WIDE_PAIR_TOWER_PLAN, n, channels, H, W, blocks, stem, sm_count)


def _wide_plan(entry, fields, n, channels, H, W, blocks, stem, sm_count):
    lib = _lib.load_library()
    out = (C.c_int64 * 9)()
    if not getattr(lib, entry)(n, channels, H, W, blocks, int(stem), sm_count, out):
        return None, lib.mz_last_error(None).decode()
    return dict(zip(fields, out)), ""


def debug_wide_tower(x, weights, biases=None, site="prediction", actions=None, A=1, parents=None, pool_stride=1, parts=1,
                     device=0):
    """One 128-channel x3 tensor-core tower of a network call site through mz_debug_wide_tower; numpy NCHW in and out.
    x is [n, 128, H, W]; ``weights`` the convs in order ([128, 129, 3, 3] dynamics stem first, then two [128, 128, 3, 3]
    per block), ``biases`` one [128] per conv.  ``site`` as for debug_conv_tower.  Returns (out [n, 128, H, W], kernel
    launches, range-guard count, the plan of the launch as a dict)."""
    return _wide_tower("mz_debug_wide_tower", WIDE_TOWER_PLAN, x, weights, biases, site, actions, A, parents, pool_stride,
                       parts, device)


def debug_wide_pair_tower(x, weights, biases=None, site="prediction", actions=None, A=1, parents=None, pool_stride=1,
                          parts=1, device=0):
    """debug_wide_tower with every board split across a CTA pair (mz_debug_wide_pair_tower), on any board the pair's
    planner accepts; the plan is a dict of WIDE_PAIR_TOWER_PLAN."""
    return _wide_tower("mz_debug_wide_pair_tower", WIDE_PAIR_TOWER_PLAN, x, weights, biases, site, actions, A, parents,
                       pool_stride, parts, device)


def _wide_tower(entry, fields, x, weights, biases, site, actions, A, parents, pool_stride, parts, device, channels=128,
                extra=()):
    """The wide debug towers' marshalling: ``extra`` are the entry's int32 arguments after pool_stride (the 256-channel
    entry's forced boards per CTA pair); the plan has len(fields) entries."""
    lib = _lib.load_library()
    _, blocks, arrays = _tower_args(x, weights, biases, site, actions, parents, channels)
    n, _, H, W = arrays[0].shape
    out = numpy.empty_like(arrays[0])
    launches, sat = C.c_int64(0), C.c_int32(0)
    plan = (C.c_int64 * len(fields))()
    rc = getattr(lib, entry)(device, n, H, W, blocks, TOWER_SITES[site], parts, A, *_ptrs(arrays), pool_stride, *extra,
                             out.ctypes.data, C.byref(launches), C.byref(sat), plan)
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    return out, launches.value, sat.value, dict(zip(fields, plan))


WIDE256_TOWER_PLAN = ("boards", "m_tiles", "threads", "smem", "stages", "layers", "ctas_per_sm", "wave", "launches", "reg_cap")


def debug_wide256_tower_plan(n, channels, H, W, blocks, stem, sm_count, boards=0):
    """Launch plan of the 256-channel x3 tensor-core tower, output channels split across a CTA pair and ``boards`` boards
    per pair (0: the largest number that fits) stacked in M (mz_debug_wide256_tower_plan, host only): (a dict of
    WIDE256_TOWER_PLAN, per-CTA figures except ``wave``, the boards per wave), "") or (None, the reason)."""
    lib = _lib.load_library()
    out = (C.c_int64 * 10)()
    if not lib.mz_debug_wide256_tower_plan(n, channels, H, W, blocks, int(stem), sm_count, boards, out):
        return None, lib.mz_last_error(None).decode()
    return dict(zip(WIDE256_TOWER_PLAN, out)), ""


def debug_wide256_tower(x, weights, biases=None, site="prediction", actions=None, A=1, parents=None, pool_stride=1, parts=1,
                        boards=0, device=0):
    """debug_wide_tower for 256 channels (mz_debug_wide256_tower): x is [n, 256, H, W], ``weights`` [256, 257, 3, 3] for a
    dynamics stem and [256, 256, 3, 3] per block conv; ``boards`` forces the boards per CTA pair (0: planned).  Returns
    (out, kernel launches, range-guard count, the plan of the launch as a dict of WIDE256_TOWER_PLAN)."""
    return _wide_tower("mz_debug_wide256_tower", WIDE256_TOWER_PLAN, x, weights, biases, site, actions, A, parents,
                       pool_stride, parts, device, channels=256, extra=(boards,))


HEADS_ROUTES = {"planned": 0, "warp": 1, "wide": 2, "generic": 3}
HEADS_ROUTE_NAMES = {1: "warp", 2: "wide", 3: "generic"}
LAYOUTS = {"dense": 0, "f16": 1, "split": 2}
HEADS_PLAN = ("route", "groups", "threads", "grid", "smem")


def _head_shapes(shapes, site):
    """int32 rows {reduced channels, logits, hidden layers, widths...} of (rc, hidden widths, n_out) head shapes."""
    want = {"representation": 0, "prediction": 2}.get(site, 1)
    if len(shapes) != want:
        raise ValueError(f"site {site} has {want} heads, got {len(shapes)}")
    rows = numpy.zeros((max(len(shapes), 1), 3 + _lib.MZ_MAX_LAYERS), numpy.int32)
    for i, (rc, hidden, n_out) in enumerate(shapes):
        if len(hidden) > _lib.MZ_MAX_LAYERS:
            raise ValueError(f"head {i}: {len(hidden)} hidden layers, at most {_lib.MZ_MAX_LAYERS}")
        rows[i, :3] = (rc, n_out, len(hidden))
        rows[i, 3:3 + len(hidden)] = hidden
    return rows


def debug_heads_plan(n, channels, H, W, heads, site, layout="dense", route="planned", g0=0, sm_count=132):
    """Launch plan of one heads call (mz_debug_heads_plan, host only): (a dict of route ("warp" = heads_kernel<32>, "wide" =
    heads_kernel<128>, "generic"), groups per CTA, threads, grid and smem, "") or (None, the reason) when the shape or the
    forced ``route`` is refused.  ``heads``: the (reduced channels, hidden widths, logits) of the site's heads - none at
    "representation", the reward head at "dynamics" / "dynamics_pool", value then policy at "prediction"."""
    lib = _lib.load_library()
    rows = _head_shapes(heads, site)
    out = (C.c_int64 * 5)()
    if not lib.mz_debug_heads_plan(n, g0, channels, H, W, TOWER_SITES[site], LAYOUTS[layout], HEADS_ROUTES[route],
                                   rows.ctypes.data, sm_count, out):
        return None, lib.mz_last_error(None).decode()
    plan = dict(zip(HEADS_PLAN, out))
    plan["route"] = HEADS_ROUTE_NAMES[plan["route"]]
    return plan, ""


def debug_heads(x, heads, site, layout="dense", route="planned", parts=1, pool_stride=1, out_slot=0, device=0):
    """The heads call of one network call site through mz_debug_heads; numpy in and out.  ``x`` [n, C, H, W] (dense; encoded
    into ``layout`` by the entry).  ``heads``: one dict per head of the site (see debug_heads_plan) with "conv_w" [rc, C],
    "conv_b" [rc] and "fc", a list of (weight [out, in], bias [out]) as in the reference state_dict.  Returns a dict: "logits"
    (one [n, n_out] per head), "scalar" [2, n], and at the rescaling sites "rescaled" [n, C, H, W], "pool" (float32
    [n, pool_stride, state floats]) and on the board layouts "state" [n, state floats]; "plan" as debug_heads_plan gives it.
    Outputs the kernels do not write keep the NaN bytes they start with."""
    lib = _lib.load_library()
    x = numpy.ascontiguousarray(x, numpy.float32)
    n, ch, H, W = x.shape
    shapes, keep, tensors = [], [], []
    for i, h in enumerate(heads):
        conv_w = numpy.ascontiguousarray(h["conv_w"], numpy.float32)
        shapes.append((conv_w.shape[0], [numpy.shape(w)[0] for w, _ in h["fc"][:-1]], numpy.shape(h["fc"][-1][0])[0]))
        named = [(f"h{i}.conv.weight", conv_w), (f"h{i}.conv.bias", h["conv_b"])]
        for l, (w, b) in enumerate(h["fc"]):
            named += [(f"h{i}.fc.{2 * l}.weight", w), (f"h{i}.fc.{2 * l}.bias", b)]
        for name, a in named:
            a = numpy.ascontiguousarray(a, numpy.float32)
            keep.append(a)
            tensors.append((name.encode(), a))
    arr = (_lib.MzTensor * max(len(tensors), 1))()
    for i, (name, a) in enumerate(tensors):
        arr[i].name, arr[i].data, arr[i].numel = name, a.ctypes.data, a.size
    rows = _head_shapes(shapes, site)
    logits = [numpy.empty((n, s[2]), numpy.float32) for s in shapes]
    scalar = numpy.empty((2, n), numpy.float32)
    pooled = site != "prediction"
    elems = ch * H * W if layout == "dense" else (2048 if layout == "f16" else 4096)
    rescaled = numpy.empty((n, ch, H, W), numpy.float32) if pooled else None
    pool = numpy.empty((n, pool_stride, elems), numpy.float32) if pooled else None
    state = numpy.empty((n, elems), numpy.float32) if pooled and layout != "dense" else None
    plan = (C.c_int64 * 5)()
    ptr = lambda a: None if a is None else a.ctypes.data        # noqa: E731
    rc = lib.mz_debug_heads(device, n, ch, H, W, TOWER_SITES[site], LAYOUTS[layout], HEADS_ROUTES[route], parts, rows.ctypes.data,
                            arr, len(tensors), x.ctypes.data, pool_stride, out_slot, ptr(logits[0] if logits else None),
                            ptr(logits[1] if len(logits) > 1 else None), scalar.ctypes.data, ptr(rescaled), ptr(pool), ptr(state),
                            plan)
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    p = dict(zip(HEADS_PLAN, plan))
    p["route"] = HEADS_ROUTE_NAMES[p["route"]]
    out = {"logits": logits, "scalar": scalar, "plan": p}
    if pooled:
        out.update(rescaled=rescaled, pool=pool)
    if state is not None:
        out["state"] = state
    return out


FC_ROUTES = {"infer_initial": 0, "infer_recurrent": 1, "infer_pool": 2, "search_root": 3, "search_sim": 4}
FC_PATH_NAMES = {0: "infer", 1: "fixed", 2: "fused", 3: "split"}
FC_NET_PLAN = ("path", "G", "threads", "grid", "smem")
H100_SMEM_OPTIN = 232448            # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KB)


def debug_fc_net_plan(spec, G, route, n, force_split=False, sm_count=132, smem_cap=H100_SMEM_OPTIN):
    """Launch plan of one fully-connected network route (mz_debug_fc_net_plan, host only) for n samples with G lanes each:
    (a dict of FC_NET_PLAN, path "infer" = fc_inference_kernel<G>, "fixed" / "fused" / "split" = the search's network call,
    "") or (None, the reason) when the shape is refused.  ``spec`` is an FC NetSpec; ``force_split`` makes the search routes
    walk the layer descriptors with the heads one after the other (the network never does)."""
    lib = _lib.load_library()
    out = (C.c_int64 * 5)()
    if not lib.mz_debug_fc_net_plan(C.byref(net_desc(spec)), spec.obs_elems, G, FC_ROUTES[route], int(force_split), n, sm_count,
                                    smem_cap, out):
        return None, lib.mz_last_error(None).decode()
    plan = dict(zip(FC_NET_PLAN, out))
    plan["path"] = FC_PATH_NAMES[plan["path"]]
    return plan, ""


def debug_fc_net(spec, weights, G, route, x, actions=None, parents=None, pool_stride=1, out_slot=0, force_split=False, device=0):
    """One fully-connected network route through mz_debug_fc_net; numpy in and out.  ``weights``: the five MLPs' tensors named
    as in the reference state_dict.  ``x``: observations [n, obs_elems] (infer_initial, search_root) or parent states [n, E];
    ``actions`` [n] on the recurrent routes; on infer_pool ``parents`` [n] is the pool slot each parent is put in and
    ``out_slot`` the slot the kernel writes.  Returns a dict of "raw" (the state before the rescale, search routes), "hidden",
    "reward_logits", "value_logits", "policy_logits", "prior", "value", "reward", "pool" (infer_pool, [n, pool_stride, E])
    and "plan" as debug_fc_net_plan gives it.  Every output starts as NaN bytes; what a route does not write keeps them."""
    lib = _lib.load_library()
    x = numpy.ascontiguousarray(x, numpy.float32)
    n = x.shape[0]
    E, A, F = spec.encoding, spec.action_space, spec.full_support
    keep, arr = [], (_lib.MzTensor * len(weights))()
    for i, (name, a) in enumerate(weights.items()):
        a = numpy.ascontiguousarray(a, numpy.float32)
        keep.append((name.encode(), a))
        arr[i].name, arr[i].data, arr[i].numel = keep[-1][0], a.ctypes.data, a.size
    out = {"raw": numpy.empty((n, E), numpy.float32), "hidden": numpy.empty((n, E), numpy.float32),
           "reward_logits": numpy.empty((n, F), numpy.float32), "value_logits": numpy.empty((n, F), numpy.float32),
           "policy_logits": numpy.empty((n, A), numpy.float32), "prior": numpy.empty((n, A), numpy.float32),
           "value": numpy.empty(n, numpy.float32), "reward": numpy.empty(n, numpy.float32)}
    pool = numpy.empty((n, pool_stride, E), numpy.float32) if route == "infer_pool" else None
    act = None if actions is None else numpy.ascontiguousarray(actions, numpy.int32)
    par = None if parents is None else numpy.ascontiguousarray(parents, numpy.int32)
    plan = (C.c_int64 * 5)()
    ptr = lambda a: None if a is None else a.ctypes.data        # noqa: E731
    rc = lib.mz_debug_fc_net(device, C.byref(net_desc(spec)), spec.obs_elems, arr, len(weights), G, FC_ROUTES[route],
                             int(force_split), n, x.ctypes.data, ptr(act), ptr(par), pool_stride, out_slot,
                             *[out[k].ctypes.data for k in ("raw", "hidden", "reward_logits", "value_logits", "policy_logits",
                                                             "prior", "value", "reward")], ptr(pool), plan)
    if rc != 0:
        raise _lib.MzError(rc, lib.mz_last_error(None).decode())
    p = dict(zip(FC_NET_PLAN, plan))
    p["path"] = FC_PATH_NAMES[p["path"]]
    out["plan"] = p
    if pool is not None:
        out["pool"] = pool
    return out
