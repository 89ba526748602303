"""Mirror of /root/reference/code/lib/model/multiply.py: the ``Multiply`` scene model whose eval-mode
``forward`` (multiply.py:174-598) drops onto the fused C-ABI entry ``mp_render_rays``.

Differences forced by the offline environment (documented in DESIGN.md):
  * the SMPL body model files are licence-gated, so SMPL servers / deformers are injected
    (``smpl_server_list``: objects with ``forward(scale, transl, thetas, betas) -> dict(smpl_verts, smpl_tfs,
    smpl_weights)`` and canonical ``verts_c``); ``scene.SyntheticSMPLServer`` is the offline stand-in;
  * ray/box hit lists (trimesh on the host in the reference, multiply.py:208-214,256) are taken from
    ``input['index_ray_box_list']`` when present, else computed on the device: against the x1.2 axis-aligned box of the
    posed vertices without any host round trip (``culling="aabb"``, default), or against the x1.2 ORIENTED box built on
    the host by ``utils/obb.py`` as the reference does with trimesh (``culling="obb"``).
"""
import numpy as np
import torch
import torch.nn as nn

from .. import engine, scene as S
from .networks import ImplicitNet, RenderingNet, _get
from .density import LaplaceDensity, AbsDensity
from .ray_sampler import ErrorBoundSampler
from .deformer import SMPLDeformer
from . import rend_util


class Multiply(nn.Module):
    def __init__(self, opt, betas_path=None, smpl_server_list=None, num_person=None, culling="aabb"):
        super().__init__()
        if culling not in ("aabb", "obb"):
            raise ValueError("culling must be 'aabb' (device-side axis-aligned box, no host round trip) or 'obb' "
                             "(oriented box on the host as in multiply.py:208-214)")
        self.culling = culling
        if smpl_server_list is None:
            raise ValueError("SMPL model files are not redistributable: pass smpl_server_list")
        self.using_nerfacc = True
        P = len(smpl_server_list) if num_person is None else num_person
        self.smpl_server_list = list(smpl_server_list)
        self.foreground_implicit_network_list = nn.ModuleList(
            [ImplicitNet(_get(opt, "implicit_network")) for _ in range(P)])
        self.foreground_rendering_network_list = nn.ModuleList(
            [RenderingNet(_get(opt, "rendering_network")) for _ in range(P)])
        self.with_bkgd = _get(opt, "with_bkgd", True)
        self.bg_implicit_network = ImplicitNet(_get(opt, "bg_implicit_network"))
        self.bg_rendering_network = RenderingNet(_get(opt, "bg_rendering_network"))
        self.frame_latent_encoder = nn.Embedding(_get(opt, "num_training_frames"), _get(opt, "dim_frame_encoding"))
        self.deformer_list = [SMPLDeformer(smpl_verts=s.verts_c, smpl_weights=s.weights, scale=getattr(s, "scale", 1.0))
                              for s in self.smpl_server_list]
        self.sdf_bounding_sphere = 3.0                                   # multiply.py:85
        self.threshold = 0.05                                            # multiply.py:88
        # canonical meshes (multiply.py:118-121): the server's triangles over its canonical vertices (mesh_verts_c when
        # the server keeps the mesh's vertices apart from verts_c, as scene.SyntheticSMPLServer does); None = no mesh
        self.mesh_v_cano_list, self.mesh_f_cano_list = [], []
        for srv in self.smpl_server_list:
            f = getattr(srv, "faces", None)
            v = getattr(srv, "mesh_verts_c", None)
            v = srv.verts_c if v is None else v
            self.mesh_v_cano_list.append(v.reshape(-1, 3) if f is not None else None)
            self.mesh_f_cano_list.append(torch.as_tensor(f).to(torch.int64) if f is not None else None)
        self._cano_meshes = {}
        d = _get(opt, "density")
        self.density = LaplaceDensity(**(dict(d) if not isinstance(d, dict) else d))
        self.bg_density = AbsDensity()
        rs = _get(opt, "ray_sampler")
        rs = dict(rs) if not isinstance(rs, dict) else dict(rs)
        rs.pop("N_samples_inverse_sphere", None)
        self.ray_sampler = ErrorBoundSampler(self.sdf_bounding_sphere, inverse_sphere_bg=True, **rs)
        self._renderer = None
        self._key = None
        self._side = {}
        self.output_buffers = None      # optional dict of preallocated output tensors (parallel.PixelBuffer.views)
        # the packed kernels are built for the shipped network shapes (confs/model/*.yaml:12,17-58): fail loudly otherwise
        fe = _get(opt, "dim_frame_encoding")
        if fe != 32:
            raise NotImplementedError("dim_frame_encoding = %r: the background chain is packed for 32" % (fe,))

    # ---- packed device state ---------------------------------------------------------------
    @property
    def field_list(self):
        return self._ensure_renderer(next(self.parameters()).device).fields

    def _scene_dict(self, persons):
        return dict(cfg=dict(self.ray_sampler.cfg, multires=6, bg_multires=10, bg_multires_view=4),
                    persons=persons,
                    bg_implicit={k: v.detach() for k, v in self.bg_implicit_network.state_dict().items()},
                    bg_render={k: v.detach() for k, v in self.bg_rendering_network.state_dict().items()},
                    frame_code=torch.zeros(1, self.frame_latent_encoder.embedding_dim),
                    beta_param=float(self.density.beta.detach()), beta_min=float(self.density.beta_min))

    def _ensure_renderer(self, device, persons=None):
        """(Re)packs the weights when a parameter changed (``_version`` counters); the per-frame state (pose, cond,
        frame code) goes through ``update_person`` / ``set_cond`` and never repacks."""
        key = (str(device), tuple(int(p._version) for p in self.parameters()))
        if self._renderer is None or self._key != key:
            if persons is None:
                persons = [self._person_dict(p, None) for p in range(len(self.smpl_server_list))]
            self._renderer = engine.Renderer(self._scene_dict(persons), device=device)
            self._key = key
            rf = getattr(self, "_root_finder", (0, 1e-5))
            if rf[0] > 0:
                for b in self._renderer.bodies:
                    b.set_root_finder(*rf)
        return self._renderer

    def set_root_finder(self, max_steps, cvg_threshold=1e-5):
        """Not in the reference (SURVEY.md §8 row f4; the reference's deformer is the closed-form inverse only):
        max_steps > 0 makes the sampler, the main pass and sdf_func_with_smpl_deformer refine every non-outlier
        canonical point with Broyden iterations on forward_skinning(x_c) = x.  0 (default) = reference behaviour."""
        self._root_finder = (int(max_steps), float(cvg_threshold))
        for d in self.deformer_list:
            d.set_root_finder(*self._root_finder)
        if self._renderer is not None:
            for b in self._renderer.bodies:
                b.set_root_finder(*self._root_finder)

    def set_render_grad(self, on=True):
        """Not in the reference's interface (the reference always back-propagates; this mirror's training forward returns
        detached values by default): on = the training forward's pixel outputs are differentiable w.r.t.
        ``density.beta`` and the per-sample sdf / rgb / normals and background sdf / rgb it exposes as
        ``res["render_samples"]`` (dict(persons=[dict(sdf, rgb, normal)], bg=dict(sdf, rgb) or None), leaf tensors whose
        ``.grad`` a network backward consumes).  ``loss.backward()`` then fills ``density.beta.grad``.  Eval mode ignores
        the switch.  Off (default) = detached values, as before."""
        self._render_grad = bool(on)

    def set_canonical_mesh(self, person_id, verts, faces):
        """Replaces person ``person_id``'s canonical mesh (verts [V,3], faces [F,3]), as multiply_model.py:504-506 does
        with the marching-cubes mesh every 20 epochs.  Its grid is rebuilt on the next use."""
        self.mesh_v_cano_list[person_id] = verts.detach().reshape(-1, 3)
        self.mesh_f_cano_list[person_id] = torch.as_tensor(faces).detach().to(torch.int64).reshape(-1, 3)
        self._cano_meshes.pop(person_id, None)

    def get_deformed_mesh_fast_mode_multiple_person(self, verts, smpl_tfs, person_id):
        """multiply.py:129-134: LBS of canonical mesh vertices verts [V,3] (or [1,V,3]) with the weights of the nearest
        canonical SMPL vertex and smpl_tfs [24,4,4] (or [1,24,4,4]) -> [1,V,3] (SMPLDeformer.forward_skinning)."""
        b = self.deformer_list[person_id].body(verts.device)
        # forward skinning reads only the canonical vertices; the posed ones keep the body's current frame
        tfs = smpl_tfs.reshape(24, 4, 4)
        b.set_pose(getattr(b, "verts_p", b.verts_c), tfs)
        if torch.is_grad_enabled() and (smpl_tfs.requires_grad or verts.requires_grad):
            xd, _ = engine.ForwardJac.apply(b, verts.reshape(-1, 3), tfs)     # differentiable in smpl_tfs (opt_depth)
            return xd[None]
        xd, _ = b.forward_jac(verts.reshape(-1, 3))
        return xd[None]

    def _canonical_mesh(self, person_id, device):
        if self.mesh_f_cano_list[person_id] is None:
            raise ValueError("person %d has no canonical mesh: the SMPL server provides no faces; call "
                             "Multiply.set_canonical_mesh(person_id, verts, faces) before training at current_epoch < 250"
                             % person_id)
        m = self._cano_meshes.get(person_id)
        if m is None or m.device != torch.device(device):
            m = engine.CanonicalMesh(self.mesh_v_cano_list[person_id], self.mesh_f_cano_list[person_id], device=device)
            self._cano_meshes[person_id] = m
        return m

    def check_off_in_surface_points_cano_mesh(self, x_cano, N_samples, person_id, threshold=0.05):
        """multiply.py:153-167: canonical points x_cano [rows*N_samples,3] against person ``person_id``'s canonical
        mesh -> (index_off_surface [rows], index_in_surface [rows]) bool: the row's minimum signed distance (negative
        inside, kaolin's check_sign) > threshold, resp. <= 0."""
        dev = x_cano.device if x_cano.is_cuda else torch.device("cuda", torch.cuda.current_device())
        return self._canonical_mesh(person_id, dev).surface_flags(x_cano, N_samples, threshold)

    def _person_dict(self, p, smpl_out, cond=None):
        srv = self.smpl_server_list[p]
        d = dict(implicit={k: v.detach() for k, v in self.foreground_implicit_network_list[p].state_dict().items()},
                 render={k: v.detach() for k, v in self.foreground_rendering_network_list[p].state_dict().items()},
                 verts_c=srv.verts_c.reshape(-1, 3), weights=srv.weights.reshape(-1, 24),
                 scale=getattr(srv, "scale", 1.0))
        if smpl_out is None:
            smpl_out = srv.canonical_output()
        d["verts_p"] = smpl_out["smpl_verts"].reshape(-1, 3)
        d["tfs"] = smpl_out["smpl_tfs"].reshape(24, 4, 4)
        d["cond"] = cond if cond is not None else torch.zeros(1, 69)
        return d

    def load_reference_checkpoint(self, state_dict, strict=True):
        """Loads a reference checkpoint: a Lightning ``ckpt['state_dict']`` (keys prefixed ``model.``,
        train.py:16-22 / multiply_model.py:81-92) or a bare ``Multiply.state_dict()``.  The reference registers
        ``smpl_server_list`` / ``deformer_list`` as ModuleLists whose SMPL modules carry the body-model buffers
        (body_models.py:152-249) and the sampler has none; those keys belong to the injected SMPL servers here and are
        dropped, as are the training-only ``body_model_list`` / ``mesh_*`` entries.  Everything else must match
        exactly when ``strict``."""
        sd = {}
        for k, v in state_dict.items():
            if k.startswith("model."):
                k = k[len("model."):]
            elif "." in k and k.split(".")[0] in ("body_model_list", "loss", "sam_server"):
                continue
            if k.split(".")[0] in ("smpl_server_list", "deformer_list", "smpl_server", "deformer", "ray_sampler",
                                   "mesh_v_cano_list", "mesh_f_cano_list", "mesh_face_vertices_list"):
                continue
            sd[k] = v
        return self.load_state_dict(sd, strict=strict)

    # ---- operator surface the sampler / callers use (multiply.py:137-151) --------------------------
    def sdf_func_with_smpl_deformer(self, x, cond, smpl_tfs, smpl_verts, person_id):
        """multiply.py:137-151: canonicalise x against person ``person_id``'s posed SMPL (nearest vertex, inverse
        LBS), evaluate the SDF network there, set outliers (> 0.1 from the body, deformer.py:49) to sdf = 4 in eval
        mode.  Returns (sdf [N,1], x_c [N,3], feature [N,256])."""
        x_c, outlier_mask = self.deformer_list[person_id].forward(x, smpl_tfs, return_weights=False, inverse=True,
                                                                  smpl_verts=smpl_verts)
        output = self.foreground_implicit_network_list[person_id](x_c, cond, person_id=person_id)[0]
        sdf = output[:, 0:1].clone()
        if not self.training:
            sdf[outlier_mask] = 4.0                                         # multiply.py:142-143
        if not self.with_bkgd and self.sdf_bounding_sphere > 0.0:
            raise NotImplementedError("with_bkgd=False (sphere clamp, multiply.py:145-148) is not on the shipped path")
        feature = output[:, 1:]
        return sdf, x_c, feature

    def _side_streams(self, dev, n):
        key = str(dev)
        if len(self._side.get(key, [])) < n:
            self._side[key] = [torch.cuda.Stream(device=dev) for _ in range(n)]
        return self._side[key][:n]

    # ---- Multiply.forward, eval branch -------------------------------------------------------
    def forward(self, input, id=-1, cond_zero_shit=False, canonical_pose=False):
        """multiply.py:174-598, eval branch.  ``id``: render only that person (``person_list = [id]``, :244-247: its
        samples alone are composited and ``acc_person_list`` is [R,1]); ``canonical_pose``: every SMPL server is
        evaluated at zero translation and the canonical hip pose (:196-201) while the pose conditioning of the
        networks still comes from ``smpl_pose`` (:270).  No host synchronisation happens on this path when the SMPL
        servers live on the device (model.smpl.SMPLServer): SMPL forward, culling, sampling, MLPs and compositing
        are all enqueued asynchronously."""
        if input["pose"].dim() == 2:            # [1,7] quaternion | centre form (rend_util.py:46-50) -> [1,4,4]
            input = dict(input, pose=rend_util.pose_matrix(input["pose"]))
        if self.training:
            return self._forward_train_values(input, id, cond_zero_shit)
        dev = input["uv"].device
        smpl_params, smpl_pose = input["smpl_params"], input["smpl_pose"]
        scale = smpl_params[:, :, 0]
        smpl_shape, smpl_trans = input["smpl_shape"], input["smpl_trans"]
        P = smpl_trans.shape[1]
        if id != -1 and not (0 <= int(id) < P):
            raise IndexError("person id %r out of range (num_person = %d)" % (id, P))
        person_list = list(range(P)) if id == -1 else [int(id)]            # multiply.py:244-247
        hits_in = input.get("index_ray_box_list")
        if hits_in is not None and len(hits_in) == P and len(person_list) != P:
            hits_in = [hits_in[i] for i in person_list]
        need_rays = hits_in is None
        if need_rays:
            dirs, cam = rend_util.get_camera_params(input["uv"], input["pose"], input["intrinsics"])
            dirs = dirs[0]
            cam = cam.expand(dirs.shape[0], 3).contiguous()
        # Per-person preparation — SMPL server, pose conditioning, posed-grid rebuild, culling — is a chain of small
        # single-CTA kernels (multiply.py:196-214, :256-263, :270).  The persons' chains are independent, so each runs on
        # its own side stream and the caller's stream waits for all of them before the render: the chains overlap
        # instead of queueing (pure stream plumbing; every kernel is the library's).
        main = torch.cuda.current_stream(dev)
        side = self._side_streams(dev, len(person_list)) if len(person_list) > 1 else [main] * len(person_list)
        start = torch.cuda.Event()
        start.record(main)
        persons = {}
        hits = []
        first_build = self._renderer is None
        if first_build:
            side = [main] * len(person_list)        # the renderer (weights) is packed on the caller's stream first

        def smpl_out(i):
            if canonical_pose:                                             # multiply.py:196-201
                cpose = torch.zeros_like(smpl_pose[:, i])
                cpose[0, 5] = np.pi / 6
                cpose[0, 8] = -np.pi / 6
                return self.smpl_server_list[i](scale[:, i], torch.zeros_like(smpl_trans[:, i]), cpose, smpl_shape[:, i])
            return self.smpl_server_list[i](scale[:, i], smpl_trans[:, i], smpl_pose[:, i], smpl_shape[:, i])

        if first_build:
            full = []
            for i in range(P):
                out = smpl_out(i)
                full.append(self._person_dict(i, out, smpl_pose[:, i, 3:] / np.pi))
            r = self._ensure_renderer(dev, full)
        else:
            r = self._ensure_renderer(dev)
        done = []
        for k, i in enumerate(person_list):
            st = side[k]
            with torch.cuda.stream(st):
                if st is not main:
                    st.wait_event(start)
                out = smpl_out(i)
                pd = dict(verts_p=out["smpl_verts"].reshape(-1, 3), tfs=out["smpl_tfs"].reshape(24, 4, 4),
                          cond=smpl_pose[:, i, 3:] / np.pi)                # multiply.py:270
                persons[i] = pd
                r.update_person(i, pd)
                if need_rays:
                    # multiply.py:208-214, :256-263: rays vs the person's box inflated by 1.2 — box, test, ordered
                    # compaction and the empty-list rule all on the device; the count stays there
                    if self.culling == "obb":
                        # the reference's choice: oriented box of the posed mesh, extents x1.2, built on the host from
                        # a device->host copy of the vertices (multiply.py:208-214); utils/obb.py restates trimesh's
                        # algorithm.  The ray test itself stays on the device.
                        from ..utils import obb
                        c, h, rot = obb.culling_box(pd["verts_p"].detach().cpu().numpy(), 1.2)
                        hits.append(engine.ray_box_hits(cam, dirs, c, h, rot, device_count=True))
                    else:
                        hits.append(engine.ray_aabb_hits(cam, dirs, pd["verts_p"], 1.2))
                if st is not main:
                    ev = torch.cuda.Event()
                    ev.record(st)
                    done.append(ev)
        for ev in done:
            main.wait_event(ev)
        if not need_rays:
            hits = hits_in
        if "image_id" in input:
            frame = self.frame_latent_encoder(input["image_id"])          # multiply.py:407-410
        elif input.get("idx") is not None:
            frame = self.frame_latent_encoder(input["idx"])
        else:
            frame = None
        if frame is not None and r.bg is not None:
            r.bg.set_cond(frame.detach())
        bg_saved = r.bg
        if frame is None:
            r.bg = None                                                    # white background, multiply.py:540-541
        try:
            ob = self.output_buffers if (self.output_buffers is not None and id == -1) else None
            out = r.render(input, hits, persons=person_list, out=ob)
        finally:
            r.bg = bg_saved
        return {k: out[k] for k in ("acc_map", "acc_person_list", "rgb_values", "fg_rgb_values", "normal_values")}

    # ---- Multiply.forward, training branch: VALUES only ------------------------------------------
    def _forward_train_values(self, input, id=-1, cond_zero_shit=False):
        """The values of the training branch of Multiply.forward (multiply.py:174-598 with self.training) for the shipped
        loss weights (smpl_surface_weight = zero_pose_weight = 0, confs/model/*.yaml:77-88): stochastic sampling with the
        reference's own random stream (the same torch.manual_seed gives the same sample depths), no outlier clamp (:142 is
        eval-only), eikonal samples and their SDF gradients (:320-331), temporal loss (:242-243), jittered background
        depths (:482).  By default NO autograd graph is built and the tensors are detached values; with
        ``set_render_grad(True)`` the pixel outputs carry the compositing stages' graph (to density.beta and the
        per-sample leaves of ``res["render_samples"]``; the networks' backward is still open, DESIGN.md 7).  One scalar read per person keeps the random stream in step with the reference's
        (its trip count decides how much randperm consumes).  At current_epoch < 250 the canonical points of the main
        pass are also tested against each person's canonical mesh (:313-316, check_off_in_surface_points_cano_mesh) and
        index_off_surface / index_in_surface [R] bool are the merged flags of :549-560; at >= 250 they are None."""
        epoch = int(input["current_epoch"])
        dev = input["uv"].device
        smpl_params, smpl_pose = input["smpl_params"], input["smpl_pose"]
        scale = smpl_params[:, :, 0]
        smpl_shape, smpl_trans = input["smpl_shape"], input["smpl_trans"]
        P = smpl_trans.shape[1]
        person_list = list(range(P)) if id == -1 else [int(id)]
        zero_cond = epoch < 20 or epoch % 20 == 0 or cond_zero_shit          # multiply.py:271-273
        dirs, cam = rend_util.get_camera_params(input["uv"], input["pose"], input["intrinsics"])
        dirs = dirs[0]
        R = dirs.shape[0]
        cam = cam.expand(R, 3).contiguous()
        hits_in = input.get("index_ray_box_list")
        persons, hits, rngs, grad_theta = {}, [], [], []
        first = self._renderer is None
        outs = {}
        for i in range(P):
            outs[i] = self.smpl_server_list[i](scale[:, i], smpl_trans[:, i], smpl_pose[:, i], smpl_shape[:, i])
        if first:
            self._ensure_renderer(dev, [self._person_dict(i, outs[i], smpl_pose[:, i, 3:] / np.pi) for i in range(P)])
        r = self._ensure_renderer(dev)
        meshes = [self._canonical_mesh(i, dev) for i in person_list] if epoch < 250 else None
        for k, i in enumerate(person_list):
            cond = smpl_pose[:, i, 3:] * 0. if zero_cond else smpl_pose[:, i, 3:] / np.pi
            pd = dict(verts_p=outs[i]["smpl_verts"].reshape(-1, 3), tfs=outs[i]["smpl_tfs"].reshape(24, 4, 4), cond=cond)
            persons[i] = pd
            r.update_person(i, pd)
            if hits_in is not None:
                h = hits_in[i] if len(hits_in) == P else hits_in[k]
            else:
                v = pd["verts_p"]
                lo, hi = v.min(0)[0], v.max(0)[0]
                h = engine.ray_box_hits(cam, dirs, ((lo + hi) / 2).tolist(), ((hi - lo) / 2 * 1.2).tolist())
            h = engine.hit_list(h, dev)
            hits.append(h)
            # the reference's draws for this person, in its order: get_z_vals (ray_sampler.py:38,171,202,212,216) ...
            rng = self.ray_sampler.draw_training_rng(h.numel())
            d, o = dirs[h].contiguous(), cam[h].contiguous()
            self.ray_sampler.get_z_vals(d, o, self, {"smpl": cond}, pd["tfs"][None], False, pd["verts_p"][None], i,
                                        rng=rng)               # decides the trip count -> the generator state
            rng = {k2: v2 for k2, v2 in rng.items() if k2 != "states"}
            rngs.append(rng)
            # ... then the eikonal samples (multiply.py:320-326): randperm(V)[:512], PointInSpace(local_sigma 0.01)
            srv = self.smpl_server_list[i]
            vc = srv.verts_c.reshape(-1, 3).to(dev)
            idx = torch.randperm(vc.shape[0])[:512].to(dev)
            sample = vc[idx] + torch.randn(1, 512, 3)[0].to(dev) * 0.01
            torch.rand(1, 0, 3)                                            # sampler.py:104-107 with global_ratio = 0
            _, _, g = r.fields[i].implicit_forward(sample, want_feat=False, want_grad=True)
            grad_theta.append(g)
        t_rand_bg = torch.rand(R, 32)                                      # multiply.py:482 (UniformSampler, training)
        if "image_id" in input:
            frame = self.frame_latent_encoder(input["image_id"])
        else:
            frame = self.frame_latent_encoder(input["idx"])
        if r.bg is not None:
            r.bg.set_cond(frame.detach())
        train = dict(rng=rngs, t_rand_bg=t_rand_bg, meshes=meshes, threshold=self.threshold)
        grad_on = getattr(self, "_render_grad", False)
        if grad_on:
            train["beta"] = self.density.get_beta()
        out = r.render(input, hits, persons=person_list, train=train)
        temporal = torch.zeros(1, device=dev)
        if epoch > 250:                                                    # multiply.py:242-243
            temporal = torch.mean(torch.square(input["smpl_pose_last"] - input["smpl_pose"])).reshape(1).detach()
        z1 = torch.zeros(1, device=dev)
        res = {"rgb_values": out["rgb_values"], "normal_values": out["normal_values"], "acc_map": out["acc_map"],
               "acc_person_list": out["acc_person_list"], "grad_theta": torch.cat(grad_theta, 0)[None],
               "index_outside": input.get("index_outside"), "index_off_surface": out.get("index_off_surface"),
               "index_in_surface": out.get("index_in_surface"),
               "interpenetration_loss": z1, "temporal_loss": temporal, "smpl_surface_loss": z1.clone(),
               "zero_pose_loss": z1.clone(), "epoch": input["current_epoch"], "cam_loc": cam,
               "t_list": [], "fg_rgb_values_each_person_list": [], "hitted_mask_idx": [], "mean_hitted_vertex_list": []}
        if grad_on:
            res["render_samples"] = dict(persons=out["samples"], bg=out.get("samples_bg"))
        if "sam_mask" in input:
            res["sam_mask"] = input["sam_mask"].squeeze()
        return res

    def query_oc(self, x, cond, person_id):
        """multiply.py:169-172: canonical SDF of person ``person_id`` at x [..., 3] under pose conditioning
        ``cond['smpl']`` [1,69] -> {'occ': [N,1]} (the mesh extractor's callback, lib/utils/mesh.py:78-132)."""
        dev = x.device
        r = self._ensure_renderer(dev)
        f = r.fields[person_id]
        c = cond["smpl"] if isinstance(cond, dict) else cond
        with torch.cuda.device(dev):
            f.set_cond(c.detach())
            sdf, _ = f.implicit_forward(x.reshape(-1, 3), want_feat=False)
        return {"occ": sdf.reshape(-1, 1)}
