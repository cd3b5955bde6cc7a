"""go1_gym_learn.ppo_cse — Runner of the reference (go1_gym_learn/ppo_cse/__init__.py:44-308) on the CUDA kernels of this repository.

`Runner(env, device).learn(num_learning_iterations, init_at_random_ep_len, eval_freq)` keeps the reference's
loop structure (24-step rollout -> compute_returns -> update -> logging/checkpoints with the same file names),
so scripts/train.py drops in unchanged.  Multi-GPU: launch one process per GPU with torchrun; each rank owns
`env.num_envs` envs, and PPO gradients / advantage statistics / KL are all-reduced over NCCL
(`Runner(..., process_group=...)` or automatically when torch.distributed is initialised)."""
import copy
import os
import time
from collections import deque

import torch
from ml_logger import logger
from params_proto import PrefixProto

from .actor_critic import ActorCritic
from .rollout_storage import RolloutStorage


def class_to_dict(obj) -> dict:
    if not hasattr(obj, "__dict__"):
        return obj
    result = {}
    for key in dir(obj):
        if key.startswith("_") or key == "terrain":
            continue
        val = getattr(obj, key)
        result[key] = [class_to_dict(i) for i in val] if isinstance(val, list) else class_to_dict(val)
    return result


class DataCaches:
    def __init__(self, curriculum_bins):
        from go1_gym_learn.ppo.metrics_caches import SlotCache, DistCache
        self.slot_cache = SlotCache(curriculum_bins)
        self.dist_cache = DistCache()


caches = DataCaches(1)


class RunnerArgs(PrefixProto, cli=False):
    # runner
    algorithm_class_name = 'RMA'
    num_steps_per_env = 24  # per iteration
    max_iterations = 1500  # number of policy updates

    # logging
    save_interval = 400  # check for potential saves every this many iterations
    save_video_interval = 100
    log_freq = 10

    # load and resume
    resume = False
    load_run = -1  # -1 = last run
    checkpoint = -1  # -1 = last saved model
    resume_path = None  # updated from load_run and chkpt
    resume_curriculum = True


class Runner:

    def __init__(self, env, device='cpu', process_group=None):
        from .ppo import PPO

        self.device = device
        self.env = env
        actor_critic = ActorCritic(self.env.num_obs, self.env.num_privileged_obs, self.env.num_obs_history,
                                   self.env.num_actions).to(self.device)

        if RunnerArgs.resume:
            # the reference downloads from a fixed MIT server (ppo_cse/__init__.py:76-82); here resume_path is a
            # local directory written by a previous run (same file names).
            weights = torch.load(os.path.join(RunnerArgs.resume_path, "checkpoints", "ac_weights_last.pt"), map_location=self.device)
            actor_critic.load_state_dict(state_dict=weights)
            if hasattr(self.env, "curricula") and RunnerArgs.resume_curriculum:
                import pickle
                p = os.path.join(RunnerArgs.resume_path, "curriculum", "distribution.pkl")
                if os.path.exists(p):
                    rows = []
                    with open(p, "rb") as f:
                        while True:
                            try:
                                rows.append(pickle.load(f))
                            except EOFError:
                                break
                    distribution_last = rows[-1]["distribution"]
                    for gait_id, gait_name in enumerate(self.env.category_names):
                        self.env.curricula[gait_id].weights = distribution_last[f"weights_{gait_name}"]

        self.alg = PPO(actor_critic, device=self.device)
        self.num_steps_per_env = RunnerArgs.num_steps_per_env
        self.alg.init_storage(self.env.num_train_envs, self.num_steps_per_env, [self.env.num_obs],
                              [self.env.num_privileged_obs], [self.env.num_obs_history], [self.env.num_actions])
        if process_group is None and torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            process_group = torch.distributed.group.WORLD
        self.process_group = process_group
        self.alg.process_group = process_group
        self.alg.storage.process_group = process_group
        if process_group is not None:       # identical initial weights on every rank
            torch.distributed.broadcast(actor_critic.flat_params, src=0, group=process_group)
            actor_critic.sample_seed = torch.distributed.get_rank(process_group)

        self.tot_timesteps = 0
        self.tot_time = 0
        self.current_learning_iteration = 0
        self.last_recording_it = 0
        self.collection_time = self.learn_time = 0.0

        self.env.reset()

    # ------------------------------------------------------------------ graph-replayed rollout
    step_graph = True       # class switch; GO1_STEP_GRAPH=0 in the environment forces the eager per-launch path

    def _step_graph_state(self):
        """Static state of the graph-replayed rollout, or None when the configuration does not allow it (eval envs, host
        curriculum, injected noise, a wrapper other than HistoryWrapper): then rollout() launches kernel by kernel."""
        st = self.__dict__.get("_sg", False)
        if st is not False:
            return st
        st = None
        env = self.env
        base = getattr(env, "env", None)
        ok = self.step_graph and os.environ.get("GO1_STEP_GRAPH", "1") != "0" and base is not None and hasattr(env, "_bufs") \
            and hasattr(base, "_device_curriculum") and self.env.num_eval_envs == 0 and self.alg.use_cuda_graph is True \
            and self.alg.actor_critic.injected_eps is None and str(self.device).startswith("cuda")
        K = len(getattr(base, "user_reward_names", ()))
        if ok and base._device_curriculum() is not None and base.cfg.commands.command_curriculum and (K == 0 or base._user_rewards_capturable()):
            from go1_b200 import capi
            dev, T = base.core.device, self.num_steps_per_env
            W = capi.NUM_EPISODE_SUMS + 1
            with torch.inference_mode(False):
                st = dict(slot=torch.zeros(1, dtype=torch.int32, device=dev), acc=torch.zeros(W, device=dev),
                          acc_hist=torch.zeros(T, W, device=dev), graphs={}, warm={0: 0, 1: 0}, W=W, T=T,
                          fork=os.environ.get("GO1_STEP_FORK", "1") != "0")
                if K:       # the user terms' extras["train/episode"] accumulator [K sums + count] and its per-step history
                    st.update(acc_user=torch.zeros(K + 1, device=dev), acc_user_hist=torch.zeros(T, K + 1, device=dev))
        self._sg = st
        return st

    def _graph_step_body(self, sg):
        """One env step of the rollout as a fixed launch sequence on static buffers (what PPO.act, LeggedRobot._step_device,
        HistoryWrapper.step and PPO.process_env_step launch, minus the per-step host logic); the storage slot, the Philox step
        counter and gravity are read from device memory, so the captured sequence serves every step."""
        import ctypes as C
        from go1_b200 import capi
        env, alg = self.env, self.alg
        base, ac, stg = env.env, alg.actor_critic, alg.storage
        core, dc, L, sp = base.core, base._dev_cur, capi.lib(), capi.stream_ptr
        hist, obs, priv = env.obs_history, core.obs, core.priv_obs
        N = core.N
        # Two independent pieces run on a side stream (forks / joins become edges of the captured graph): the periodic command resample of
        # this step beside the policy evaluation (it writes commands and curriculum state, the policy reads histories), and the storage of
        # the transition beside the history roll (both only read what the kernels before them produced; the roll writes the other buffer).
        fork = sg.get("fork", True) and (not dc.shared or os.environ.get("GO1_STEP_FORK_SHARED", "1") != "0")
        main = torch.cuda.current_stream()
        side = sg.get("side") if fork else None
        if fork and side is None:
            side = sg["side"] = torch.cuda.Stream()
        if fork:
            e0 = torch.cuda.Event(); e0.record(main)
            with torch.cuda.stream(side):
                side.wait_event(e0)
                dc.resample(1)
                e1 = torch.cuda.Event(); e1.record(side)
        actions, values = alg._act_eager(hist, priv)
        capi.check(L.go1_rollout_store_observations(capi.ptr(obs), capi.ptr(priv) if core.num_priv else None, capi.ptr(stg.observations),
                                                    capi.ptr(stg.privileged_observations) if core.num_priv else None, capi.ptr(sg["slot"]), N,
                                                    core.num_obs, core.num_priv, sp()), "go1_rollout_store_observations")
        if fork:
            main.wait_event(e1)
        else:
            dc.resample(1)
        base._raw_actions = actions           # user reward terms read env.actions: this step's, from the tensor the graph writes
        base._sim_step(actions, 0)
        dc.gather()
        sg["acc"].zero_()
        dc.resample(0)
        dc.reset_envs(actions, True, 0, sg["acc"])
        if "acc_user" in sg:
            core.user_reward_fold(dc.out_ids, dc.out_count, 0, base._user_sums, None, sg["acc_user"], sg["acc_user_hist"], sg["slot"])
        if fork:
            e2 = torch.cuda.Event(); e2.record(main)
        else:
            env._roll(core.obs)
        send_to = bool(base.cfg.env.send_timeouts)
        h16 = ac.model_inputs.get("act") if stg.hist_bf16 else None       # a BF16 slab stores the BF16 history the policy just evaluated
        assert h16 is not None or not stg.hist_bf16
        ins = [None, None, None if stg.hist_bf16 else hist, actions, core.rew, values, ac._logp, ac._mean, ac.std.data, dc.env_bins_f32]
        outs = [stg.observations, stg.privileged_observations, stg.observation_histories, stg.actions, stg.rewards, stg.values, stg.actions_log_prob,
                stg.mu, stg.sigma, stg.env_bins]
        for x in ins[3:]:
            assert x.is_contiguous() and x.dtype == torch.float32
        assert stg.hist_bf16 or (stg.history_rows_fit(hist) and hist.dtype == torch.float32)      # the store copies whole rows at the slab's pitch
        from .ppo import PPO_Args

        def store_and_advance():
            capi.check(L.go1_rollout_store_transition((C.c_void_p * 10)(*[x.data_ptr() if x is not None else None for x in ins]), capi.ptr(core.reset_u8),
                                                      capi.ptr(dc.time_outs_u8) if send_to else None, (C.c_void_p * 10)(*[x.data_ptr() for x in outs]),
                                                      capi.ptr(stg.dones), capi.ptr(sg["slot"]), N, core.num_obs, core.num_priv, stg.hist_row_pitch,
                                                      actions.shape[1], float(PPO_Args.gamma), sp()), "go1_rollout_store_transition")
            if h16 is not None:
                capi.check(L.go1_rollout_store_rows_bf16(capi.ptr(h16), h16.stride(0), capi.ptr(stg._hist_slab), stg.hist_row_pitch, capi.ptr(sg["slot"]),
                                                         N, h16.shape[1], sp()), "go1_rollout_store_rows_bf16")
            capi.check(L.go1_rollout_advance(capi.ptr(sg["acc"]), capi.ptr(sg["acc_hist"]), sg["W"], sg["T"], capi.ptr(sg["slot"]), capi.ptr(core.step_dev), sp()),
                       "go1_rollout_advance")

        if fork:
            with torch.cuda.stream(side):
                side.wait_event(e2)
                store_and_advance()
                e3 = torch.cuda.Event(); e3.record(side)
            env._roll(core.obs)
            main.wait_event(e3)
        else:
            store_and_advance()
        return actions

    def _rollout_graphed(self, sg):
        """The 24-step collection phase as CUDA-graph replays: one graph per parity of the history ping-pong buffers; the first
        two steps of either parity run eagerly (they are ordinary steps of the rollout), the third is captured."""
        from go1_b200 import capi
        from go1_gym.envs.base.legged_robot import _LazyDict
        env, alg = self.env, self.alg
        base, ac = env.env, alg.actor_critic
        core, dc, L = base.core, base._dev_cur, capi.lib()
        if base._ep_len_dirty:
            base._sync_interval_events_after_ep_len_write()
        dc.to_device()
        sg["slot"].zero_()
        core.step_dev.fill_(base.common_step_counter + 1)
        with torch.inference_mode():
            for i in range(self.num_steps_per_env):
                p = env._cur
                key = (p, ac.flat_params.data_ptr())
                g = sg["graphs"].get(key)
                if g is None and sg["warm"][p] < 2:
                    sg["warm"][p] += 1
                    actions = self._graph_step_body(sg)
                elif g is None and any(k[1] != key[1] for k in sg["graphs"]):
                    # the flat weight buffer was rebuilt (ActorCritic.to()): drop the graphs captured against the old one and warm up again
                    # (the eager steps also rebuild the packed weight copies the new graphs will read)
                    sg["graphs"].clear()
                    sg["warm"] = {0: 0, 1: 0}
                    sg["warm"][p] += 1
                    actions = self._graph_step_body(sg)
                elif g is None:
                    graph = torch.cuda.CUDAGraph()
                    ac.ensure_packed()
                    cap = {}
                    if ac.deterministic:    # captured on a stream of its own whose workspace (go1_set_deterministic) is sized before the capture
                        cap["stream"] = self.__dict__.setdefault("_det_capture_stream", torch.cuda.Stream())
                        capi.check(L.go1_deterministic_reserve(cap["stream"].cuda_stream), "go1_deterministic_reserve")
                    n0 = L.go1_kernel_launch_count()
                    with torch.cuda.graph(graph, **cap):
                        actions = self._graph_step_body(sg)
                    n_kernels = L.go1_kernel_launch_count() - n0
                    L.go1_kernel_launch_add(-n_kernels)
                    env._cur = p; env.obs_history = env._bufs[p]       # capture ran the host half of _roll without executing anything
                    g = sg["graphs"][key] = (graph, actions, n_kernels)
                if g is not None:
                    graph, actions, n_kernels = g
                    ac.ensure_packed()                                 # packed weight copies are refreshed once per weight version, outside the graph
                    graph.replay()
                    L.go1_kernel_launch_add(n_kernels)
                    env._cur = p ^ 1; env.obs_history = env._bufs[p ^ 1]
                base._raw_actions = actions
                base.common_step_counter += 1
                base._post_physics_step_callback_host()
        core.step_dev.zero_()
        alg.storage.step = self.num_steps_per_env
        alg.transition.clear()
        # extras / metrics of the whole rollout from ONE snapshot of the per-step accumulators
        acc_hist = sg["acc_hist"].clone()
        base._episode_acc_prev = acc_hist[-1]
        user_hist = sg["acc_user_hist"].clone() if "acc_user_hist" in sg else [None] * self.num_steps_per_env
        if "acc_user_hist" in sg:
            base._user_acc_prev = user_hist[-1]
        ex = base.extras
        ex["train/episode"] = _LazyDict(base._episode_builder(acc_hist[-1], may_be_empty=True, user_acc=user_hist[-1]))
        ex["env_bins"] = dc.env_bins_f32
        ex["curriculum/distribution"] = _LazyDict(base._distribution_builder())
        if base.cfg.env.send_timeouts:
            ex["time_outs"] = dc.time_outs
        ex["privileged_obs"] = core.priv_obs
        if hasattr(logger, "store_metrics_lazy"):
            for t in range(self.num_steps_per_env):
                logger.store_metrics_lazy('train/episode', _LazyDict(base._episode_builder(acc_hist[t], may_be_empty=True, user_acc=user_hist[t])))
        return core.obs, core.priv_obs, env.obs_history, ex

    def rollout(self, obs, privileged_obs, obs_history, eval_expert=False):
        """The 24-step collection phase of learn() (ppo_cse/__init__.py:138-187)."""
        sg = self._step_graph_state()
        if sg is not None and obs_history is self.env.obs_history and self.env.env._dev_cur is not None:
            try:
                return self._rollout_graphed(sg)
            except Exception as e:          # capture not possible in this context: same kernels, launched one by one
                if sg["graphs"] or any(sg["warm"].values()):
                    raise
                print(f"[go1_b200] graph-replayed rollout disabled: {type(e).__name__}: {e}")
                self._sg = None
        num_train_envs = self.env.num_train_envs
        infos = {}
        with torch.inference_mode():
            for i in range(self.num_steps_per_env):
                actions_train = self.alg.act(obs[:num_train_envs], privileged_obs[:num_train_envs], obs_history[:num_train_envs])
                if self.env.num_eval_envs > 0:
                    if eval_expert:
                        actions_eval = self.alg.actor_critic.act_teacher(obs_history[num_train_envs:], privileged_obs[num_train_envs:])
                    else:
                        actions_eval = self.alg.actor_critic.act_student(obs_history[num_train_envs:])
                    actions = torch.cat((actions_train, actions_eval), dim=0)
                else:
                    actions = actions_train
                obs_dict, rewards, dones, infos = self.env.step(actions)
                obs, privileged_obs, obs_history = obs_dict["obs"], obs_dict["privileged_obs"], obs_dict["obs_history"]
                self.alg.process_env_step(rewards[:num_train_envs], dones[:num_train_envs], infos)
                for key in ('train/episode', 'eval/episode'):
                    if key in infos:
                        if hasattr(logger, "store_metrics_lazy"):      # expanded once per log_metrics_summary, not per env step
                            logger.store_metrics_lazy(key, infos[key])
                        else:
                            with logger.Prefix(metrics=key):
                                logger.store_metrics(**infos[key])
        return obs, privileged_obs, obs_history, infos

    def learn(self, num_learning_iterations, init_at_random_ep_len=False, eval_freq=100, curriculum_dump_freq=500, eval_expert=False):
        from ml_logger import logger
        assert logger.prefix, "you will overwrite the entire instrument server"
        logger.start('start', 'epoch', 'episode', 'run', 'step')

        if init_at_random_ep_len:
            self.env.episode_length_buf = torch.randint_like(self.env.episode_length_buf, high=int(self.env.max_episode_length))

        num_train_envs = self.env.num_train_envs
        obs_dict = self.env.get_observations()
        obs, privileged_obs, obs_history = obs_dict["obs"], obs_dict["privileged_obs"], obs_dict["obs_history"]
        self.alg.actor_critic.train()

        rank0 = self.process_group is None or torch.distributed.get_rank(self.process_group) == 0
        tot_iter = self.current_learning_iteration + num_learning_iterations
        it = self.current_learning_iteration
        for it in range(self.current_learning_iteration, tot_iter):
            start = time.time()
            obs, privileged_obs, obs_history, infos = self.rollout(obs, privileged_obs, obs_history, eval_expert)
            distribution = infos.get('curriculum/distribution')
            stop = time.time()
            self.collection_time = stop - start
            start = stop
            with torch.inference_mode():
                self.alg.compute_returns(obs_history[:num_train_envs], privileged_obs[:num_train_envs])
            if it % curriculum_dump_freq == 0 and rank0:
                logger.save_pkl({"iteration": it, **caches.slot_cache.get_summary(), **caches.dist_cache.get_summary()},
                                path=f"curriculum/info.pkl", append=True)
                if distribution is not None:
                    logger.save_pkl({"iteration": it, "distribution": distribution}, path=f"curriculum/distribution.pkl", append=True)

            (mean_value_loss, mean_surrogate_loss, mean_adaptation_module_loss, mean_decoder_loss, mean_decoder_loss_student,
             mean_adaptation_module_test_loss, mean_decoder_test_loss, mean_decoder_test_loss_student) = self.alg.update()
            self.learn_time = time.time() - start

            logger.store_metrics(
                time_elapsed=logger.since('start'), time_iter=logger.split('epoch'),
                adaptation_loss=mean_adaptation_module_loss, mean_value_loss=mean_value_loss,
                mean_surrogate_loss=mean_surrogate_loss, mean_decoder_loss=mean_decoder_loss,
                mean_decoder_loss_student=mean_decoder_loss_student, mean_decoder_test_loss=mean_decoder_test_loss,
                mean_decoder_test_loss_student=mean_decoder_test_loss_student,
                mean_adaptation_module_test_loss=mean_adaptation_module_test_loss)

            if RunnerArgs.save_video_interval:
                self.log_video(it)

            world = 1 if self.process_group is None else torch.distributed.get_world_size(self.process_group)
            self.tot_timesteps += self.num_steps_per_env * self.env.num_envs * world
            if logger.every(RunnerArgs.log_freq, "iteration", start_on=1) and rank0:
                logger.log_metrics_summary(key_values={"timesteps": self.tot_timesteps, "iterations": it})
                logger.job_running()

            if it % RunnerArgs.save_interval == 0 and rank0:
                self.save(it)
            self.current_learning_iteration += num_learning_iterations
        if rank0:
            self.save(it)

    def save(self, it):
        """Same artefacts as the reference (ppo_cse/__init__.py:231-274): ac_weights_{it:06d}.pt (+ _last), and
        TorchScript exports of the adaptation module and actor body for go1_gym_deploy."""
        with logger.Sync():
            logger.torch_save(self.alg.actor_critic.state_dict(), f"checkpoints/ac_weights_{it:06d}.pt")
            logger.duplicate(f"checkpoints/ac_weights_{it:06d}.pt", f"checkpoints/ac_weights_last.pt")
            path = './tmp/legged_data'
            os.makedirs(path, exist_ok=True)
            adaptation_module_path = f'{path}/adaptation_module_latest.jit'
            adaptation_module = copy.deepcopy(self.alg.actor_critic.adaptation_module).to('cpu')
            torch.jit.script(adaptation_module).save(adaptation_module_path)
            body_path = f'{path}/body_latest.jit'
            body_model = copy.deepcopy(self.alg.actor_critic.actor_body).to('cpu')
            torch.jit.script(body_model).save(body_path)
            logger.upload_file(file_path=adaptation_module_path, target_path=f"checkpoints/", once=False)
            logger.upload_file(file_path=body_path, target_path=f"checkpoints/", once=False)

    def log_video(self, it):
        if it - self.last_recording_it >= RunnerArgs.save_video_interval:
            self.env.start_recording()
            if self.env.num_eval_envs > 0:
                self.env.start_recording_eval()
            self.last_recording_it = it
        frames = self.env.get_complete_frames()
        if len(frames) > 0:
            self.env.pause_recording()
            logger.save_video(frames, f"videos/{it:05d}.mp4", fps=1 / self.env.dt)
        if self.env.num_eval_envs > 0:
            frames = self.env.get_complete_frames_eval()
            if len(frames) > 0:
                self.env.pause_recording_eval()
                logger.save_video(frames, f"videos/{it:05d}_eval.mp4", fps=1 / self.env.dt)

    def get_inference_policy(self, device=None):
        self.alg.actor_critic.eval()
        if device is not None:
            self.alg.actor_critic.to(device)
        return self.alg.actor_critic.act_inference

    def get_expert_policy(self, device=None):
        self.alg.actor_critic.eval()
        if device is not None:
            self.alg.actor_critic.to(device)
        return self.alg.actor_critic.act_expert
