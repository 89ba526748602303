"""Ray-block sharding over the GPUs of one box (SURVEY.md §8e).

Rays are independent except for the sampler's batch-global convergence flag, so the path shards with
no data-path collective: rank g renders the contiguous block [g*R/G, (g+1)*R/G) and one all-gather
assembles the pixel records.  Parity is defined per shard (a shard is exactly a smaller batch of
the reference)."""
import torch
import torch.distributed as dist

from . import _lib as L, engine
from .model import rend_util

PIXEL_KEYS = ("rgb_values", "fg_rgb_values", "normal_values", "acc_map", "acc_person_list")


def shard_bounds(total, rank, world):
    """Contiguous, balanced ray blocks: the first (total % world) ranks get one extra ray."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_inputs(inputs, rank, world):
    lo, hi = shard_bounds(inputs["uv"].shape[1], rank, world)
    out = dict(inputs)
    out["uv"] = inputs["uv"][:, lo:hi].contiguous()
    return out, (lo, hi)


def pack_pixels(out):
    """[R_local, 3+3+3+1+P] record per ray."""
    return torch.cat([out["rgb_values"], out["fg_rgb_values"], out["normal_values"], out["acc_map"][:, None],
                      out["acc_person_list"]], dim=1).contiguous()


def unpack_pixels(rec, P):
    return {"rgb_values": rec[:, 0:3], "fg_rgb_values": rec[:, 3:6], "normal_values": rec[:, 6:9],
            "acc_map": rec[:, 9], "acc_person_list": rec[:, 10:10 + P]}


class PixelBuffer:
    """The pixel record of a ray block as ONE flat device buffer [rgb R*3 | fg_rgb R*3 | normal R*3 | acc R |
    acc_person R*P]; the renderer writes its outputs straight into the views (``Renderer.render(out=buf.views)``) and
    a single all_gather_into_tensor of ``flat`` assembles the frame — no concatenation kernel in between."""

    def __init__(self, R, P, device):
        self.R, self.P = R, P
        self.flat = torch.empty(R * (10 + P), device=device)
        o = [0, 3 * R, 6 * R, 9 * R, 10 * R, (10 + P) * R]
        f = self.flat
        self.views = {"rgb_values": f[o[0]:o[1]].view(R, 3), "fg_rgb_values": f[o[1]:o[2]].view(R, 3),
                      "normal_values": f[o[2]:o[3]].view(R, 3), "acc_map": f[o[3]:o[4]],
                      "acc_person_list": f[o[4]:o[5]].view(R, P)}

    @staticmethod
    def frame(gathered, world, R, P):
        """gathered [world, R*(10+P)] -> dict of full-frame tensors [world*R, ...] (copies: the blocks are strided)."""
        g = gathered.view(world, -1)
        cut = lambda a, b, w: g[:, a * R:b * R].reshape(world * R, w) if w > 1 else g[:, a * R:b * R].reshape(world * R)
        return {"rgb_values": cut(0, 3, 3), "fg_rgb_values": cut(3, 6, 3), "normal_values": cut(6, 9, 3),
                "acc_map": cut(9, 10, 1), "acc_person_list": g[:, 10 * R:(10 + P) * R].reshape(world * R, P)}


def gather_pixels(out, total, group=None):
    """All-gather the per-rank pixel records into the full frame (every rank gets it).  Blocks may differ by
    one ray, so records are padded to the largest block for the collective."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rec = pack_pixels(out)
    P = out["acc_person_list"].shape[1]
    if world == 1:
        return unpack_pixels(rec, P)
    sizes = [shard_bounds(total, r, world) for r in range(world)]
    mx = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros(mx, rec.shape[1], device=rec.device, dtype=rec.dtype)
    pad[: rec.shape[0]] = rec
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    full = torch.cat([b[: hi - lo] for b, (lo, hi) in zip(bufs, sizes)], dim=0)
    return unpack_pixels(full, P)


# ---------------------------------------------------------------------------------------------------------------
# Person-sharded rendering (SURVEY.md §8e row 2, BASELINE configs[4]): one canonical field per GPU.
#
#   1. rank owner(p) holds person p's body + MLP weights and produces p's per-ray sample lists for ALL rays of the
#      call (sampler -> deformer -> SDF / normals / colour): rows [R_p, 8n+1] = z_vals (n+1) | sdf (n) | rgb (3n) |
#      normal (3n), in hit-list order.  The sampler's batch-global flag (ray_sampler.py:137) therefore sees exactly the
#      rays it sees in the single-GPU forward.
#   2. ONE exchange: the compositor needs every person's samples of a ray together, so the rows of the rays of block b
#      travel to rank b (hit lists are sorted -> a block is a contiguous row range; all ranks know all ranges).
#   3. rank b composites its block (mp_composite), renders the block's background, composes the pixels.
#   4. the usual all-gather of pixel records.
# The result is bit-identical to Renderer.render on one GPU (tests/test_gpu_person_shard.py).
# ---------------------------------------------------------------------------------------------------------------
def person_owner(p, world):
    return p % world


def normalize_hits(hit_lists):
    """engine.hit_list of every person's ray ids, left where they are (multiply.py:262-263: empty -> ray 0)."""
    return [engine.hit_list(h) for h in hit_lists]


def exchange_plan(hit_lists, total_rays, world):
    """plan[p][b] = (lo, hi): rows of person p's (sorted) hit list whose ray ids fall in ray block b."""
    plan = []
    for h in hit_lists:
        h = h.cpu()
        edges = torch.tensor([shard_bounds(total_rays, b, world)[0] for b in range(world)] + [total_rays])
        cut = torch.searchsorted(h, edges).tolist()
        plan.append([(cut[b], cut[b + 1]) for b in range(world)])
    return plan


def _global_rank(group, r):
    """P2POp peers are GLOBAL ranks; `r` is a rank of `group`."""
    return r if group is None else dist.get_global_rank(group, r)


def exchange_person_rows(rows, plan, width, rank, world, device, group=None):
    """rows: {p: [R_p, width] tensor} for the persons this rank owns.  Returns {p: [cnt_p, width]} for every person:
    the rows of this rank's ray block.  One batch of point-to-point transfers (the all-to-all by ray block)."""
    P = len(plan)
    got = {}
    ops = []
    for p in range(P):
        own = person_owner(p, world)
        lo, hi = plan[p][rank]
        if own == rank:
            got[p] = rows[p][lo:hi]
            for b in range(world):
                blo, bhi = plan[p][b]
                if b != rank and bhi > blo:
                    ops.append(dist.P2POp(dist.isend, rows[p][blo:bhi].contiguous(), _global_rank(group, b), group))
        else:
            got[p] = torch.empty(hi - lo, width, device=device, dtype=torch.float32)
            if hi > lo:
                ops.append(dist.P2POp(dist.irecv, got[p], _global_rank(group, own), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return got


class PersonShardedRenderer:
    """Eval forward with the persons' fields sharded over the ranks of the default process group."""

    def __init__(self, scene, device="cuda", group=None):
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.device = torch.device(device)
        self.scene = scene
        self.P = len(scene["persons"])
        self.cfg = scene["cfg"]
        self.n = engine.samples_per_ray(self.cfg)
        self.width = 8 * self.n + 1
        self.mine = [p for p in range(self.P) if person_owner(p, self.world) == self.rank]
        # this rank's persons only; no background in the per-person pass
        sub = dict(scene)
        sub["persons"] = [scene["persons"][p] for p in self.mine]
        sub["bg_implicit"] = None
        sub["bg_render"] = None
        self.sub = engine.Renderer(sub, device=device) if self.mine else None
        self.bg = None
        if scene.get("bg_implicit") is not None:
            self.bg = engine.Field(scene["bg_implicit"], scene["bg_render"], background=True, device=device)
            self.bg.set_cond(scene["frame_code"])
        self.beta = engine.sampler_beta(scene["beta_param"], scene.get("beta_min", engine.BETA_MIN))

    def person_rows(self, inputs, hits):
        """Step 1: [R_p, 8n+1] rows of the persons this rank owns."""
        rows = {}
        if not self.mine:
            return rows
        o = self.sub.render(inputs, [hits[p] for p in self.mine], debug=True)
        for k, p in enumerate(self.mine):
            Rp = hits[p].numel()
            rows[p] = torch.cat([o[f"z_vals_{k}"], o[f"sdf_{k}"], o[f"rgb_{k}"].reshape(Rp, -1),
                                 o[f"normals_{k}"].reshape(Rp, -1)], dim=1).contiguous()
        return rows

    def composite_block(self, inputs, hits, got, lo, hi):
        """Step 3 for the ray block [lo, hi)."""
        dev = self.device
        n, Rb = self.n, hi - lo
        keep = []
        for p in range(self.P):
            r = got[p]
            cnt = r.shape[0]
            rlo, rhi = self._plan[p][self.rank]
            idx = (hits[p][rlo:rhi].to(dev) - lo).contiguous()
            z = r[:, : n + 1].contiguous()
            sdf = r[:, n + 1: 2 * n + 1].contiguous()
            rgb = r[:, 2 * n + 1: 5 * n + 1].contiguous()
            nrm = r[:, 5 * n + 1: 8 * n + 1].contiguous()
            if cnt == 0:      # valid (never dereferenced) pointers for an empty person
                idx = torch.zeros(1, dtype=torch.int64, device=dev)
                z = sdf = rgb = nrm = torch.zeros(1, device=dev)
            keep.append((idx, z, sdf, rgb, nrm, cnt))
        persons = engine.person_samples(keep)
        fg = torch.empty(Rb, 3, device=dev)
        out = {"rgb_values": torch.empty(Rb, 3, device=dev), "fg_rgb_values": torch.empty(Rb, 3, device=dev),
               "normal_values": torch.empty(Rb, 3, device=dev), "acc_map": torch.empty(Rb, device=dev),
               "acc_person_list": torch.empty(Rb, self.P, device=dev)}
        bgT = torch.empty(Rb, device=dev)
        if Rb == 0:
            return out
        ws = L.workspace(L.call("mp_composite_workspace_bytes", Rb, self.P), dev)
        L.call("mp_composite", persons, self.P, Rb, n, self.beta, fg, out["normal_values"], out["acc_map"],
               out["acc_person_list"], bgT, ws, ws.numel())
        bg = None
        if self.bg is not None:
            uv = L.dev(inputs["uv"].reshape(-1, 2)[lo:hi], dev)
            dirs, cam = rend_util.camera_rays(uv, inputs["pose"], inputs["intrinsics"])
            bg = self.bg.bg_pixels(dirs, cam, self.cfg["scene_bounding_sphere"])
            keep += [uv, dirs, cam]
        L.call("mp_final_compose", fg, bgT, bg, Rb, out["rgb_values"], out["fg_rgb_values"])
        self._keep = keep + [fg, bgT, bg, ws]
        return out

    def render(self, inputs, hit_lists):
        """Full frame on every rank: the dict of Multiply.forward (multiply.py:589-598)."""
        hits = normalize_hits(hit_lists)
        R = inputs["uv"].reshape(-1, 2).shape[0]
        self._plan = exchange_plan(hits, R, self.world)
        rows = self.person_rows(inputs, hits)
        if self.world > 1:
            got = exchange_person_rows(rows, self._plan, self.width, self.rank, self.world, self.device, self.group)
        else:
            got = rows
        lo, hi = shard_bounds(R, self.rank, self.world)
        out = self.composite_block(inputs, hits, got, lo, hi)
        return gather_pixels(out, R, self.group)
