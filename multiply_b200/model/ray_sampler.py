"""Mirror of /root/reference/code/lib/model/ray_sampler.py (ErrorBoundSampler, eval mode)."""
import torch

from .. import _lib as L
from .. import engine


class ErrorBoundSampler:
    """ray_sampler.py:45-230.  Same constructor; ``get_z_vals`` keeps the reference's signature and return
    shape ``((z_vals, z_vals_bg), z_samples_eik)`` and runs the whole Algorithm-1 loop on the device
    (mp_sample_rays) without a host synchronisation."""

    def __init__(self, scene_bounding_sphere, near, N_samples, N_samples_eval, N_samples_extra, eps, beta_iters,
                 max_total_iters, inverse_sphere_bg=False, N_samples_inverse_sphere=0, add_tiny=0.0):
        if not inverse_sphere_bg:
            raise NotImplementedError("the reference always builds the sampler with inverse_sphere_bg=True "
                                      "(multiply.py:92)")
        self.cfg = dict(scene_bounding_sphere=scene_bounding_sphere, near=near, N_samples=N_samples,
                        N_samples_eval=N_samples_eval, N_samples_extra=N_samples_extra, eps=eps,
                        beta_iters=beta_iters, max_total_iters=max_total_iters, add_tiny=add_tiny)
        self.scene_bounding_sphere = scene_bounding_sphere
        self.N_samples, self.N_samples_eval, self.N_samples_extra = N_samples, N_samples_eval, N_samples_extra
        self._ws = None
        self.last_trips = None

    def get_z_vals(self, ray_dirs, cam_loc, model, cond, smpl_tfs, eval_mode, smpl_verts, person_id, rng=None):
        """model: object exposing ``density`` (LaplaceDensity), ``deformer_list`` and ``field_list`` —
        model.multiply.Multiply does."""
        training = bool(getattr(model, "training", False))
        dev = ray_dirs.device
        R = ray_dirs.shape[0]
        c = engine.sampler_cfg(self.cfg, float(model.density.beta.detach()), float(model.density.beta_min))
        body = model.deformer_list[person_id].body(dev)
        body.set_pose(smpl_verts[0], smpl_tfs[0] if smpl_tfs.ndim == 4 else smpl_tfs)
        field = model.field_list[person_id]
        field.set_cond(cond["smpl"])
        z = torch.empty(R, engine.samples_per_ray(self.cfg) + 1, device=dev)
        z_bg = torch.empty(R, 32, device=dev)
        trips = torch.zeros(1, dtype=torch.int32, device=dev)
        need = L.call("mp_sampler_workspace_bytes", c, R)
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = L.workspace(need, dev)
        d, o = L.dev(ray_dirs, dev), L.dev(cam_loc, dev)
        if training:
            return self._get_z_vals_training(L.lib(), c, body, field, d, o, R, z, z_bg, trips, dev, rng=rng)
        L.call("mp_sample_rays", c, body.handle, field.handle, d, o, R, z, z_bg, trips, self._ws, self._ws.numel())
        self.last_trips = trips
        # z_samples_eik only feeds the training-time eikonal term (ray_sampler.py:211-213)
        return (z, z_bg), z[:, :1]

    def draw_training_rng(self, R):
        """The reference's random draws of one training-mode get_z_vals call, from torch's global CPU generator in the
        reference's order (ray_sampler.py:38 rand(R,E) -> :171 rand(R,S) -> :202 randperm(M) -> :212 randint -> :38 again
        for the inverse-sphere sampler, rand(R,32)).  M = trips * E is only known on the device, so the draws that follow
        the loop are made for EVERY possible trip count from the same generator state; ``states[t]`` is the generator
        state the reference would be left in after t+1 trips."""
        E, S, X = self.N_samples_eval, self.N_samples, self.N_samples_extra
        T = int(self.cfg["max_total_iters"])
        t_rand = torch.rand(R, E)
        u_final = torch.rand(R, S)
        base = torch.get_rng_state()
        perm = torch.zeros(T, T * E, dtype=torch.int32)
        eik = torch.zeros(T, R, dtype=torch.int32)
        bg = torch.zeros(T, R, 32)
        states = []
        for t in range(T):
            torch.set_rng_state(base)
            if X > 0:
                perm[t, :(t + 1) * E] = torch.randperm((t + 1) * E).to(torch.int32)
            eik[t] = torch.randint(S + X + 2, (R,)).to(torch.int32)
            bg[t] = torch.rand(R, 32)
            states.append(torch.get_rng_state())
        torch.set_rng_state(base)
        return dict(t_rand=t_rand, u_final=u_final, extra_perm=perm, eik_idx=eik, t_rand_bg=bg, states=states)

    def _get_z_vals_training(self, lib, c, body, field, d, o, R, z, z_bg, trips, dev, rng=None):
        """model.training: stochastic sampling (ray_sampler.py:32-40,171,202,212-218) with the reference's own random
        stream — the same torch.manual_seed gives the same sample depths as the reference."""
        if rng is None:
            rng = self.draw_training_rng(R)
        r, dv = engine.sampler_rng_struct(rng, dev)
        z_eik = torch.empty(R, device=dev)
        L.call("mp_sample_rays_train", c, body.handle, field.handle, d, o, R, r, z, z_bg, z_eik, trips, self._ws,
               self._ws.numel())
        self.last_trips = trips
        if "states" in rng:
            # leave the generator where the reference would be: after the draws of the trip count the loop took
            # (one scalar read; the reference itself synchronises every trip, ray_sampler.py:137)
            torch.set_rng_state(rng["states"][int(trips.item()) - 1])
        self._keep = dv
        return (z, z_bg), z_eik[:, None]
