"""RolloutStorage of ppo_cse (reference go1_gym_learn/ppo_cse/rollout_storage.py:5-178): [T, N, .] slabs,
GAE through the warp-scan kernel, minibatches through the row-gather kernel."""
import torch

from go1_b200 import capi
from .actor_critic import AC_Args, history_kmajor, in_mode


class RolloutStorage:
    class Transition:
        def __init__(self):
            self.observations = None
            self.privileged_observations = None
            self.observation_histories = None
            self.critic_observations = None
            self.actions = None
            self.rewards = None
            self.dones = None
            self.values = None
            self.actions_log_prob = None
            self.action_mean = None
            self.action_sigma = None
            self.env_bins = None
            self.history_bf16 = None      # AC_Args.gemm_impl = 2: the BF16 history the policy evaluated (ActorCritic.model_inputs["act"])

        def clear(self):
            self.__init__()

    def __init__(self, num_envs, num_transitions_per_env, obs_shape, privileged_obs_shape, obs_history_shape, actions_shape, device='cpu'):
        self.device = device
        self.obs_shape, self.privileged_obs_shape = obs_shape, privileged_obs_shape
        self.obs_history_shape, self.actions_shape = obs_history_shape, actions_shape
        T, N = num_transitions_per_env, num_envs
        z = lambda *s, **k: torch.zeros(T, N, *s, device=self.device, **k)
        self.observations = z(*obs_shape)
        self.privileged_observations = z(*privileged_obs_shape)
        # the history slab [T][N][hist_row_pitch] (the pitch of HistoryWrapper's rows, capi.history_pitch) and its [T][N][K0] view.
        # AC_Args.gemm_impl = 2: BF16 rows at capi.bf16_pitch (half the bytes), holding exactly the BF16 history the policy evaluated
        K0 = int(obs_history_shape[-1])
        self.hist_bf16 = int(AC_Args.gemm_impl) == 2
        self.hist_row_pitch = capi.bf16_pitch(K0) if self.hist_bf16 else capi.history_pitch(K0)
        self._hist_slab = z(self.hist_row_pitch, dtype=torch.bfloat16) if self.hist_bf16 else z(self.hist_row_pitch)
        self.observation_histories = self._hist_slab[..., :K0]
        # Row pitch of the GATHERED minibatch histories: a multiple of 32 floats, so that every 128-byte row of a TMA box of the first-layer
        # products starts on a 128-byte line.  Measured (tools/epi_bench.py): the 24576 x 1280 x 2100 product runs in 180 us with a
        # 2112-float pitch against 259 us with the natural 2100 (each misaligned box row costs a fifth L2 sector).
        self.hist_pitch = (K0 + 31) // 32 * 32
        self.rewards = z(1)
        self.actions = z(*actions_shape)
        self.dones = z(1).byte()
        self.actions_log_prob = z(1)
        self.values = z(1)
        self.returns = z(1)
        self.advantages = z(1)
        self.mu = z(*actions_shape)
        self.sigma = z(*actions_shape)
        self.env_bins = z(1)
        self.num_transitions_per_env, self.num_envs = T, N
        self.step = 0
        self._stats = torch.zeros(2, dtype=torch.float64, device=self.device)
        self.process_group = None          # set by the multi-GPU runner: advantage statistics are global

    def add_transitions(self, transition: Transition):
        if self.step >= self.num_transitions_per_env:
            raise AssertionError("Rollout buffer overflow")
        t = self.step
        self.observations[t].copy_(transition.observations)
        self.privileged_observations[t].copy_(transition.privileged_observations)
        self.observation_histories[t].copy_(transition.observation_histories)
        self.actions[t].copy_(transition.actions)
        self.rewards[t].copy_(transition.rewards.view(-1, 1))
        self.dones[t].copy_(transition.dones.view(-1, 1))
        self.values[t].copy_(transition.values)
        self.actions_log_prob[t].copy_(transition.actions_log_prob.view(-1, 1))
        self.mu[t].copy_(transition.action_mean)
        self.sigma[t].copy_(transition.action_sigma)
        self.env_bins[t].copy_(transition.env_bins.view(-1, 1))
        self.step += 1

    def snapshot_observations(self, obs, privileged_obs):
        """Copy the observations the policy acts on into slot `step` NOW.  The env writes its next observations into the same
        buffers during env.step, so a reference kept until process_env_step would store s_{t+1} next to a_t (the reference is
        safe only because its compute_observations allocates fresh tensors).  Returns the two storage views."""
        if self.step >= self.num_transitions_per_env:
            raise AssertionError("Rollout buffer overflow")
        t = self.step
        so, sp = self.observations[t], self.privileged_observations[t]
        if obs.is_cuda and obs.dtype == torch.float32 and obs.is_contiguous() and privileged_obs.dtype == torch.float32 and privileged_obs.is_contiguous():
            capi.check(capi.lib().go1_store_observations(capi.ptr(obs), capi.ptr(privileged_obs) if sp.shape[-1] else None, capi.ptr(so),
                                                         capi.ptr(sp) if sp.shape[-1] else None, self.num_envs, so.shape[-1], sp.shape[-1],
                                                         capi.stream_ptr()), "go1_store_observations")
        else:
            so.copy_(obs); sp.copy_(privileged_obs)
        return so, sp

    def history_rows_fit(self, h):
        """The fused transition store copies whole hist_row_pitch-wide rows: h [N][K0] qualifies if it is contiguous (pitch K0) or, for a
        padded pitch, has exactly that row stride over storage that holds every full row (HistoryWrapper's buffers).  A BF16 slab takes
        its rows from the policy's BF16 input instead (add_transitions_fused)."""
        if self.hist_bf16:
            return True
        P = self.hist_row_pitch
        if P == h.shape[-1]:
            return h.is_contiguous()
        return h.dim() == 2 and h.stride(1) == 1 and h.stride(0) == P and h.untyped_storage().nbytes() >= 4 * (h.storage_offset() + h.shape[0] * P)

    def add_transitions_fused(self, tr, time_outs, gamma):
        """add_transitions + the time-out bootstrap in ONE kernel (go1_store_transition)."""
        import ctypes as C
        if self.step >= self.num_transitions_per_env:
            raise AssertionError("Rollout buffer overflow")
        t = self.step
        u8 = lambda x: x if x.dtype == torch.uint8 else (x.view(torch.uint8) if x.dtype == torch.bool else x.to(torch.uint8))
        dones, touts = u8(tr.dones), (u8(time_outs) if time_outs is not None else None)
        stored = lambda x, slot: None if (x is None or x.data_ptr() == slot.data_ptr()) else x       # already snapshotted by act()
        h16 = tr.history_bf16 if self.hist_bf16 else None
        assert not self.hist_bf16 or (h16 is not None and h16.dtype == torch.bfloat16 and h16.shape[0] == self.num_envs), \
            "a BF16 history slab stores the BF16 history the policy evaluated (PPO.act at AC_Args.gemm_impl = 2)"
        ins = [stored(tr.observations, self.observations[t]), stored(tr.privileged_observations, self.privileged_observations[t]),
               None if self.hist_bf16 else tr.observation_histories, tr.actions, tr.rewards, tr.values, tr.actions_log_prob, tr.action_mean, tr.action_sigma_vec, tr.env_bins]
        outs = [self.observations[t], self.privileged_observations[t], self.observation_histories[t], self.actions[t], self.rewards[t], self.values[t],
                self.actions_log_prob[t], self.mu[t], self.sigma[t], self.env_bins[t]]
        for k, x in enumerate(ins):
            assert x is None or ((self.history_rows_fit(x) if k == 2 else x.is_contiguous()) and x.dtype == torch.float32 and x.is_cuda), \
                "transition tensors must be contiguous float32 CUDA tensors (histories: rows at hist_row_pitch)"
        assert tr.env_bins.numel() == self.num_envs and dones.numel() == self.num_envs
        arr_in = (C.c_void_p * 10)(*[x.data_ptr() if x is not None else None for x in ins])
        arr_out = (C.c_void_p * 10)(*[x.data_ptr() for x in outs])
        capi.check(capi.lib().go1_store_transition(arr_in, capi.ptr(dones), capi.ptr(touts), arr_out, capi.ptr(self.dones[t]), self.num_envs,
                                                   self.observations.shape[-1], self.privileged_observations.shape[-1], self.hist_row_pitch,
                                                   self.actions.shape[-1], float(gamma), capi.stream_ptr()), "go1_store_transition")
        if h16 is not None:
            capi.check(capi.lib().go1_rollout_store_rows_bf16(capi.ptr(h16), h16.stride(0), capi.ptr(self._hist_slab[t]), self.hist_row_pitch, None,
                                                              self.num_envs, h16.shape[1], capi.stream_ptr()), "go1_rollout_store_rows_bf16")
        self.step += 1

    def clear(self):
        self.step = 0

    deterministic = False       # the learner's mode (AC_Args.deterministic), set by PPO.init_storage

    @in_mode
    def compute_returns(self, last_values, gamma, lam):
        T, N = self.num_transitions_per_env, self.num_envs
        L, st = capi.lib(), capi.stream_ptr()
        last_values = last_values.contiguous()
        capi.check(L.go1_ppo_gae(capi.ptr(self.rewards), capi.ptr(self.dones), capi.ptr(self.values), capi.ptr(last_values),
                                 capi.ptr(self.returns), capi.ptr(self.advantages), capi.ptr(self._stats), T, N, float(gamma), float(lam), st), "gae")
        count = T * N
        if self.process_group is not None:
            import torch.distributed as dist
            dist.all_reduce(self._stats, group=self.process_group)
            count = T * N * dist.get_world_size(self.process_group)
        capi.check(L.go1_ppo_normalize_advantages(capi.ptr(self.advantages), capi.ptr(self._stats), count, T * N, st), "normalize")

    def get_statistics(self):
        done = self.dones
        done[-1] = 1
        flat_dones = done.permute(1, 0, 2).reshape(-1, 1)
        done_indices = torch.cat((flat_dones.new_tensor([-1], dtype=torch.int64), flat_dones.nonzero(as_tuple=False)[:, 0]))
        trajectory_lengths = (done_indices[1:] - done_indices[:-1])
        return trajectory_lengths.float().mean(), self.rewards.mean()

    def gather(self, src, idx, out=None, ldd=None, key=None):
        """out[i] = src.flatten(0,1)[idx[i]] through go1_gather_rows (destination buffers are reused across updates)."""
        flat = src.flatten(0, 1)
        assert idx.dtype == torch.int64 and idx.is_contiguous() and flat.dtype == torch.float32
        w = flat.shape[1]
        ldd = ldd or w
        if out is None and key is not None:
            out = self._buffer(key, (idx.shape[0], ldd), torch.float32)
        if out is None:
            out = torch.empty(idx.shape[0], ldd, device=flat.device)
        capi.check(capi.lib().go1_gather_rows(capi.ptr(flat), capi.ptr(idx), capi.ptr(out), idx.shape[0], w, ldd, capi.stream_ptr()), "gather")
        return out if ldd == w else out[:, :w]

    def _buffer(self, key, shape, dtype):
        """A destination buffer kept across updates (reallocated when the minibatch shape changes)."""
        cache = self.__dict__.setdefault("_gather_bufs", {})
        out = cache.get(key)
        if out is None or out.shape != shape or out.dtype != dtype:
            out = cache[key] = torch.empty(*shape, device=self.device, dtype=dtype)
        return out

    def mini_batch_generator(self, num_mini_batches, num_epochs=8, indices=None):
        batch_size = self.num_envs * self.num_transitions_per_env
        mini_batch_size = batch_size // num_mini_batches
        if indices is None:
            indices = torch.randperm(num_mini_batches * mini_batch_size, requires_grad=False, device=self.device)
        dones8 = None
        bf16 = self.hist_bf16
        if bf16 != (int(AC_Args.gemm_impl) == 2):
            raise capi.Go1Error("RolloutStorage keeps its history slab in the precision of the AC_Args.gemm_impl it was built under: "
                                "build the storage again (PPO.init_storage) after changing the mode")
        for epoch in range(num_epochs):
            for i in range(num_mini_batches):
                idx = indices[i * mini_batch_size:(i + 1) * mini_batch_size].contiguous()
                obs = self.gather(self.observations, idx)
                priv_b = self.gather(self.privileged_observations, idx)
                K0, P, M = self.observation_histories.shape[-1], priv_b.shape[1], idx.shape[0]
                if bf16:    # AC_Args.gemm_impl = 2: the minibatch history, copied from the BF16 slab, and its K-major copy in BF16
                    hist_b = self._buffer(("hist16", i), (M, capi.bf16_pitch(K0)), torch.bfloat16)[:, :K0]
                    kmajor = (K0 + 1 + 2 * P, capi.bf16_pitch(M)), torch.bfloat16
                    capi.check(capi.lib().go1_gather_rows_bf16(capi.ptr(self._hist_slab), self.hist_row_pitch, capi.ptr(idx), capi.ptr(hist_b),
                                                               hist_b.stride(0), M, K0, capi.stream_ptr()), "gather_rows_bf16")
                else:
                    # whole slab rows: go1_gather_rows reads its source at a row pitch equal to the width it copies
                    hist_b = self.gather(self._hist_slab, idx, key=("hist", i), ldd=self.hist_pitch)[:, :K0]
                    kmajor = (K0 + 1 + 2 * P, (M + 31) // 32 * 32), torch.float32
                # its K-major transpose [history | 1 | priv | latent rows] for the first layers' weight-gradient products, built once per
                # update and read by every epoch (ActorCritic.backward_ppo / backward_adaptation); 830 MB for 4 minibatches at 4096 envs in fp32
                hist_b.hT = history_kmajor(hist_b, priv_b, self._buffer(("histT", i), *kmajor))
                yield (obs, obs, priv_b, hist_b,
                       self.gather(self.actions, idx), self.gather(self.values, idx), self.gather(self.advantages, idx),
                       self.gather(self.returns, idx), self.gather(self.actions_log_prob, idx), self.gather(self.mu, idx),
                       self.gather(self.sigma, idx), dones8, self.gather(self.env_bins, idx))
