"""PPO of ppo_cse (reference go1_gym_learn/ppo_cse/ppo.py:13-205) on explicit kernels: fused loss+gradient
kernel, hand-written MLP backward, one global grad-norm + clip + Adam launch over the flat parameter buffer,
device-side adaptive-KL learning rate (no per-minibatch host sync), optional NCCL gradient all-reduce."""
import torch

from go1_b200 import capi
from go1_gym_learn.ppo_cse import ActorCritic
from go1_gym_learn.ppo_cse import RolloutStorage
from go1_gym_learn.ppo_cse import caches
from go1_gym_learn.ppo_cse.actor_critic import _Net, in_mode
from params_proto import PrefixProto


class PPO_Args(PrefixProto):
    # algorithm
    value_loss_coef = 1.0
    use_clipped_value_loss = True
    clip_param = 0.2
    entropy_coef = 0.01
    num_learning_epochs = 5
    num_mini_batches = 4  # mini batch size = num_envs*nsteps / nminibatches
    learning_rate = 1.e-3  # 5.e-4
    adaptation_module_learning_rate = 1.e-3
    num_adaptation_module_substeps = 1
    schedule = 'adaptive'  # could be adaptive, fixed
    gamma = 0.99
    lam = 0.95
    desired_kl = 0.01
    max_grad_norm = 1.

    selective_adaptation_module_loss = False


class _FlatAdam:
    """torch.optim.Adam semantics (betas .9/.999, eps 1e-8) over a slice of the flat buffer."""

    def __init__(self, ac, start, end, lr):
        self.ac, self.start, self.end, self.lr = ac, start, end, lr
        n = end - start
        dev = ac.flat_params.device
        self.exp_avg = torch.zeros(n, device=dev)
        self.exp_avg_sq = torch.zeros(n, device=dev)
        self.t = 0
        self.param_groups = [{"lr": lr}]

    def step(self, grad_sq=None, max_norm=0.0, lr_dev=None):
        self.t += 1
        p = self.ac.flat_params[self.start:self.end]
        g = self.ac.flat_grads[self.start:self.end]
        capi.check(capi.lib().go1_ppo_adam_step(capi.ptr(p), capi.ptr(g), capi.ptr(self.exp_avg), capi.ptr(self.exp_avg_sq), self.end - self.start,
                                                capi.ptr(grad_sq) if grad_sq is not None else None, float(max_norm), float(self.param_groups[0]["lr"]),
                                                capi.ptr(lr_dev) if lr_dev is not None else None, 0.9, 0.999, 1e-8, self.t, capi.stream_ptr()), "adam")
        self.ac.weights_version += 1


class PPO:
    actor_critic: ActorCritic

    def __init__(self, actor_critic, device='cpu'):
        self.device = device
        self.actor_critic = actor_critic
        self.actor_critic.to(device)
        self.actor_critic.flatten()
        self.storage = None  # initialized later
        ac = self.actor_critic
        self.optimizer = _FlatAdam(ac, ac.HEAD, ac.n_params, PPO_Args.learning_rate)
        # the reference builds a second Adam over ALL parameters (ppo.py:45-46); only the adaptation module ever
        # receives a non-zero gradient from it, so its state is kept for that slice only (identical updates).
        self.adaptation_module_optimizer = _FlatAdam(ac, ac.HEAD, ac.n_adapt_params, PPO_Args.adaptation_module_learning_rate)
        self.transition = RolloutStorage.Transition()
        self.learning_rate = PPO_Args.learning_rate
        dev = ac.flat_params.device
        self._lr_dev = torch.full((1,), PPO_Args.learning_rate, device=dev)
        self._grad_sq = torch.zeros(1, dtype=torch.float64, device=dev)
        self._dstd = torch.zeros(ac.num_actions, device=dev)
        self._acc = torch.zeros(6, device=dev)
        self.process_group = None          # set by the multi-GPU runner
        self.fixed_minibatch_indices = None  # parity tests inject the permutation

    # the loss scalars live in the head of the flat gradient buffer and ride in the gradient all-reduce
    _scalars = property(lambda self: self.actor_critic.flat_grads[0:8])
    _mse_scalars = property(lambda self: self.actor_critic.flat_grads[8:10])

    deterministic = property(lambda self: self.actor_critic.deterministic)      # the mode of in_mode: the ActorCritic's

    def init_storage(self, num_envs, num_transitions_per_env, actor_obs_shape, privileged_obs_shape, obs_history_shape, action_shape):
        self.storage = RolloutStorage(num_envs, num_transitions_per_env, actor_obs_shape, privileged_obs_shape, obs_history_shape, action_shape, self.device)
        self.storage.deterministic = self.actor_critic.deterministic

    def test_mode(self):
        self.actor_critic.eval()

    def train_mode(self):
        self.actor_critic.train()

    use_cuda_graph = True      # rollout policy evaluation (11 GEMMs + sampling) replayed as one CUDA graph

    def _act_eager(self, obs_history, privileged_obs):
        actions, values = self.actor_critic.act_and_evaluate(obs_history, privileged_obs)
        return actions.detach(), values.detach()

    _MAX_INPLACE_GRAPHS = 4

    def _act_graphed(self, obs_history, privileged_obs):
        """Same computation through a captured CUDA graph with static outputs and a device-side RNG counter.  The history
        wrapper ping-pongs between two buffers and the privileged observations live in one, so a graph is captured per
        input address and reads its inputs in place (no 34 MB staging copy per step); callers that keep passing fresh
        tensors fall back to one graph with static input copies."""
        ac = self.actor_critic
        st = self.__dict__.setdefault("_graph_state", {})
        key = (obs_history.shape[0], ac._impl(), obs_history.data_ptr(), privileged_obs.data_ptr(), ac.flat_params.data_ptr())
        for stale in [k2 for k2 in st if k2[4] != key[4]]:      # graphs captured against a flat weight buffer that was rebuilt (.to())
            del st[stale]
        g = st.get(key)
        if g is None:
            # in place: contiguous histories, and rows at a TMA-readable pitch (HistoryWrapper's padded rows, capi.history_pitch)
            h_rows = obs_history.is_contiguous() or (obs_history.dim() == 2 and obs_history.stride(1) == 1 and
                                                     _Net._tma_ok(obs_history, obs_history.stride(0)))
            inplace = h_rows and privileged_obs.is_contiguous() and sum(1 for k2 in st if k2[2] is not None) < self._MAX_INPLACE_GRAPHS
            if not inplace:
                key = (obs_history.shape[0], ac._impl(), None, None, ac.flat_params.data_ptr())
                g = st.get(key)
        if g is None:
            if inplace:
                h_in, p_in = obs_history, privileged_obs          # keeps the two tensors alive for the graph's lifetime
            else:
                with torch.inference_mode(False):
                    h_in = torch.empty_like(obs_history); p_in = torch.empty_like(privileged_obs)
                h_in.copy_(obs_history); p_in.copy_(privileged_obs)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    self._act_eager(h_in, p_in)             # allocates every scratch buffer, configures kernels
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            ac.ensure_packed()                                    # the graph reads the packed weight copies, it does not build them
            L = capi.lib()
            n0 = L.go1_kernel_launch_count()
            # deterministic mode: captured on the stream of the warm-up calls, whose workspace (go1_set_deterministic) they have sized
            with torch.cuda.graph(graph, **({"stream": side} if ac.deterministic else {})):
                outs = self._act_eager(h_in, p_in)
            n_kernels = L.go1_kernel_launch_count() - n0          # this library's kernels inside the graph
            L.go1_kernel_launch_add(-n_kernels)                   # capture launched nothing
            g = st[key] = (graph, h_in, p_in, outs, (ac._mean, ac._logp, ac._last_actions, ac._value, ac._latent), inplace, n_kernels)
        graph, h_in, p_in, outs, attrs, inplace, n_kernels = g
        if not inplace:
            h_in.copy_(obs_history); p_in.copy_(privileged_obs)
        ac.ensure_packed()
        graph.replay()
        capi.lib().go1_kernel_launch_add(n_kernels)
        ac._mean, ac._logp, ac._last_actions, ac._value, ac._latent = attrs     # the graph's static outputs
        return outs

    @in_mode
    def act(self, obs, privileged_obs, obs_history):
        tr = self.transition
        ac = self.actor_critic
        if self.use_cuda_graph and obs_history.is_cuda and ac.injected_eps is None and self.use_cuda_graph != "failed":
            try:
                tr.actions, tr.values = self._act_graphed(obs_history, privileged_obs)
            except Exception as e:      # capture not possible in this context: fall back to eager launches of the same kernels
                print(f"[go1_b200] CUDA graph capture of PPO.act disabled: {type(e).__name__}: {e}")
                PPO.use_cuda_graph = "failed"
                tr.actions, tr.values = self._act_eager(obs_history, privileged_obs)
        else:
            tr.actions, tr.values = self._act_eager(obs_history, privileged_obs)
        tr.actions_log_prob = self.actor_critic.get_actions_log_prob(tr.actions).detach()
        tr.action_mean = self.actor_critic.action_mean.detach()
        tr.action_sigma = self.actor_critic.action_std.detach()
        # obs / privileged_obs are views of buffers the next env.step overwrites in place: snapshot them into the storage slot now
        tr.observations, tr.privileged_observations = self.storage.snapshot_observations(obs, privileged_obs)
        tr.critic_observations = tr.observations
        tr.observation_histories = obs_history
        if self.storage.hist_bf16:    # the BF16 slab stores what the policy evaluated
            tr.history_bf16 = self.actor_critic.model_inputs.get("act")
        return tr.actions

    def process_env_step(self, rewards, dones, infos):
        tr = self.transition
        tr.dones = dones
        tr.env_bins = infos["env_bins"]
        f32 = lambda x: x.is_cuda and x.is_contiguous() and x.dtype == torch.float32
        h = tr.observation_histories
        fused = f32(rewards) and h.is_cuda and h.dtype == torch.float32 and self.storage.history_rows_fit(h) and f32(tr.env_bins) and f32(tr.values) and \
            tr.env_bins.numel() == rewards.numel() and (not self.storage.hist_bf16 or tr.history_bf16 is not None)
        if fused:   # rewards += gamma * values * time_outs (ppo.py:84-86) happens inside the store kernel
            tr.rewards = rewards
            tr.action_sigma_vec = self.actor_critic.std.data
            self.storage.add_transitions_fused(tr, infos.get('time_outs'), PPO_Args.gamma)
        else:
            tr.rewards = rewards.clone()
            if 'time_outs' in infos:
                tr.rewards += PPO_Args.gamma * torch.squeeze(tr.values * infos['time_outs'].unsqueeze(1).to(self.device), 1)
            self.storage.add_transitions(tr)
        tr.clear()
        self.actor_critic.reset(dones)

    @in_mode
    def compute_returns(self, last_critic_obs, last_critic_privileged_obs):
        last_values = self.actor_critic.evaluate(last_critic_obs, last_critic_privileged_obs, tag="last").detach()
        self.storage.compute_returns(last_values, PPO_Args.gamma, PPO_Args.lam)

    def _allreduce(self, t):
        if self.process_group is not None:
            import torch.distributed as dist
            dist.all_reduce(t, group=self.process_group)

    @in_mode
    def update(self):
        ac, L, st = self.actor_critic, capi.lib(), capi.stream_ptr
        world = 1
        if self.process_group is not None:
            import torch.distributed as dist
            world = dist.get_world_size(self.process_group)
        self._acc.zero_()
        self._lr_dev.fill_(self.learning_rate)
        n_updates = 0
        # The reference draws ONE permutation per update and reuses it for all epochs (rollout_storage.py:101), so the
        # gathered minibatches are built once and reused.
        batches = list(self.storage.mini_batch_generator(PPO_Args.num_mini_batches, 1, indices=self.fixed_minibatch_indices))
        for it_mb in range(PPO_Args.num_learning_epochs * len(batches)):
            bi = it_mb % len(batches)
            (obs_b, critic_obs_b, priv_b, hist_b, actions_b, target_values_b, adv_b, returns_b, old_logp_b, old_mu_b, old_sigma_b, masks_b, env_bins_b) = batches[bi]
            M = hist_b.shape[0]
            mean_b, value_b = ac.forward_all(hist_b, priv_b, tag="train")
            dmean = ac._nets["actor"]._buf(("train", "dmean"), M, ac.num_actions)
            dvalue = ac._nets["critic"]._buf(("train", "dvalue"), M, 1)
            capi.check(L.go1_ppo_loss(capi.ptr(mean_b), mean_b.stride(0), capi.ptr(ac.std.data), capi.ptr(value_b), capi.ptr(actions_b), capi.ptr(old_logp_b),
                                      capi.ptr(old_mu_b), capi.ptr(old_sigma_b), capi.ptr(adv_b), capi.ptr(returns_b), capi.ptr(target_values_b),
                                      capi.ptr(dmean), ac.num_actions, capi.ptr(dvalue), capi.ptr(self._dstd), capi.ptr(self._scalars), M, ac.num_actions,
                                      PPO_Args.clip_param, PPO_Args.value_loss_coef, PPO_Args.entropy_coef, int(PPO_Args.use_clipped_value_loss),
                                      1.0 / (M * world), st()), "ppo_loss")
            ac.backward_ppo(hist_b, priv_b, dmean, dvalue, self._dstd, hT=getattr(hist_b, "hT", None))
            # ONE collective per optimizer step: gradients (already scaled by 1/global batch) + the 8 loss scalars in the buffer head
            self._allreduce(ac.flat_grads)
            if PPO_Args.desired_kl is not None and PPO_Args.schedule == 'adaptive':   # ppo.py:118-132, on the device, from the global KL
                capi.check(L.go1_ppo_adaptive_lr(capi.ptr(self._scalars), capi.ptr(self._lr_dev), PPO_Args.desired_kl, 1e-5, 1e-2, st()), "adaptive_lr")
            capi.check(L.go1_ppo_grad_sqnorm(capi.ptr(ac.flat_grads[ac.HEAD:]), ac.n_params - ac.HEAD, capi.ptr(self._grad_sq), st()), "sqnorm")
            self.optimizer.step(self._grad_sq, PPO_Args.max_grad_norm, self._lr_dev)
            self._acc[0:2] += self._scalars[0:2]

            num_train = int(M // 5 * 4)
            for epoch in range(PPO_Args.num_adaptation_module_substeps):
                outs = ac.adaptation_forward(hist_b)
                pred = outs[-1]
                dpred = ac._nets["adapt"]._buf(("adapt", "dpred"), M, pred.shape[1])
                # selective_adaptation_module_loss: train and test MSE of privileged column 0 only (ppo.py:177-183)
                dim = 1 if PPO_Args.selective_adaptation_module_loss else pred.shape[1]
                if dim < pred.shape[1]:
                    dpred[:, dim:].zero_()
                capi.check(L.go1_ppo_mse(capi.ptr(pred), pred.stride(0), capi.ptr(priv_b), priv_b.stride(0), capi.ptr(dpred), dpred.stride(0),
                                         capi.ptr(self._mse_scalars), M, num_train, dim, st()), "mse")
                ac.backward_adaptation(hist_b, outs, dpred, hT=getattr(hist_b, "hT", None))
                if self.process_group is not None:      # adaptation gradients + the MSE pair (buffer head) in one averaging all-reduce
                    import torch.distributed as dist
                    dist.all_reduce(ac.flat_grads[:ac.n_adapt_params], op=dist.ReduceOp.AVG, group=self.process_group)
                self.adaptation_module_optimizer.step()
                self._acc[2:4] += self._mse_scalars
            n_updates += 1

        acc = self._acc.tolist()                      # the only host sync of the update
        self.learning_rate = float(self._lr_dev.item())
        self.optimizer.param_groups[0]["lr"] = self.learning_rate
        num_updates = PPO_Args.num_learning_epochs * PPO_Args.num_mini_batches
        sub = num_updates * PPO_Args.num_adaptation_module_substeps
        mean_value_loss = acc[1] / num_updates
        mean_surrogate_loss = acc[0] / num_updates
        mean_adaptation_module_loss = acc[2] / sub
        mean_adaptation_module_test_loss = acc[3] / sub
        self.storage.clear()
        return mean_value_loss, mean_surrogate_loss, mean_adaptation_module_loss, 0.0, 0.0, mean_adaptation_module_test_loss, 0.0, 0.0
