"""The body of the reference's training loop (train.py:80-252) on the gif_b200 modules: one D step + one G step per
iteration, R1 every 16th iteration (train.py:145-149), optional path-length regularisation (train.py:205-208, adopted
rule), Adam with the reference's hyper-parameters (train.py:365-382), EMA of the generator (train.py:250).

Differences from the reference, all deliberate (SURVEY 3.2 / 8e):
  * nn.DataParallel -> FlatGradAllReducer (one all-reduce per net per step);
  * ONE generator forward per iteration instead of two (three with PPL).  The reference calls the generator in the D step
    (train.py:157, result detached at :160) and again in the G step (train.py:197) with the same inputs while the
    generator's weights are unchanged (only D is updated in between), so both calls return bit-identical images; the
    path-length term differentiates the same images w.r.t. the same w.  Here the forward runs once with a graph: the D
    step consumes ``fake.detach()``, the G step (and PPL) reuse the graph.  Same arithmetic, one third of the G forwards;
  * data loading / FID / checkpoints are outside the hot path.
"""
import copy
import math

import torch
import torch.nn.functional as F

from . import losses
from .distributed import FlatGradAllReducer
from .model.stg2_discriminator import Discriminator
from .model.stg2_generator import StyledGenerator


def world_gt1(reducer):
    return reducer.world > 1


def requires_grad(model, flag=True):
    """my_utils/generic_utils.py:58-60."""
    for p in model.parameters():
        p.requires_grad = flag


def accumulate(model1, model2, decay=0.999):
    """my_utils/generic_utils.py:63-76 (EMA), as one fused foreach update.  Written under no_grad rather than through
    ``.data``, so that the parameters' version counters (which the prepared-weight cache keys on) see the write."""
    with torch.no_grad():
        p1, p2 = list(model1.parameters()), list(model2.parameters())
        torch._foreach_mul_(p1, decay)
        torch._foreach_add_(p1, p2, alpha=1 - decay)


class GifTrainer:
    def __init__(self, device, resolution=256, vocab=70_000, r1_every=16, ppl=False, world_size=1, seed=0,
                 texture_loss=False, embedding_reg_weight=0.0, adaptive_interp_loss=False):
        torch.manual_seed(seed)
        self.device = device
        self.step_idx = int(math.log2(resolution)) - 2                           # train.py:387
        self.generator = StyledGenerator(embedding_vocab_size=vocab, rendered_flame_ascondition=True,
                                         normal_maps_as_cond=True, core_tensor_res=4, n_mlp=8).to(device)
        self.discriminator = Discriminator(resolution, num_color_chnls=9, channel_multiplier=2).to(device)
        self.g_running = copy.deepcopy(self.generator).train(False)
        g_ratio, d_ratio = 4 / 5, 16 / 17                                        # train.py:365-366
        # torch.optim.Adam with the step as multi-tensor CUDA launches and the step counter on the device (CUDA graphs)
        from .optim import FusedAdam
        self.g_optimizer = FusedAdam(self.generator.parameters(), lr=0.002 * g_ratio, betas=(0.0, 0.99 ** g_ratio))
        self.d_optimizer = FusedAdam(self.discriminator.parameters(), lr=0.002 * d_ratio, betas=(0.0, 0.99 ** d_ratio))
        self.g_reducer = FlatGradAllReducer(list(self.generator.parameters()), world_size)
        self.d_reducer = FlatGradAllReducer(list(self.discriminator.parameters()), world_size)
        self.r1_every = r1_every
        self.embedding_reg_weight = float(embedding_reg_weight)      # train.py:216-219 (0 in every shipped configuration)
        self.adaptive_interp_loss = bool(adaptive_interp_loss)       # train.py:236-237
        self.ppl = losses.PathLengthRegularizor() if ppl else None
        self.iteration = 0
        self._graphs = None
        self.vocab = vocab
        # texture_loss: False | True (per-GPU batch 32) | the per-GPU batch size (max_images_in_batch, train.py:59-60)
        self.interp_tex_loss = self._build_texture_loss(device, 32 if texture_loss is True else int(texture_loss)) if texture_loss else None
        requires_grad(self.generator, False)

    def _build_texture_loss(self, device, max_images_in_batch):
        """train.py:57-60 + 224-238 (apply_texture_space_interpolation_loss, enabled in the flagship run,
        configurations.py:217): FLAME decoder, condition renderer, texture space and the pairwise loss, all on the device.
        The licence-gated model files are replaced by the synthetic FLAME-shaped model (gif_b200/flame_synth.py)."""
        from .flame import FLAME
        from .flame_synth import flame_uv, synthetic_flame_model, synthetic_flame_params, synthetic_texture_data
        from .render import FlameRenderer
        from .texture_space import FlameTextureSpace, InterpolatedTextureLoss
        flame = FLAME.from_arrays(synthetic_flame_model()).to(device)
        uv, uvf = flame_uv()
        renderer = FlameRenderer(flame.faces_tensor.cpu(), uv, uvf, image_size=256).to(device)
        _, _, albedo, lights = synthetic_flame_params(1, seed=0)
        albedo, lights = albedo.to(device), lights.to(device)

        def render_condition(flame_batch):          # losses.py:186-221 (159-parameter layout): texture render + normal map
            n = flame_batch.shape[0]
            verts, _ = flame.decode_vertices(flame_batch[:, :100].float(), flame_batch[:, 100:150].float(),
                                             flame_batch[:, 150:156].float())
            return renderer.render_tex_and_normal(verts, flame_batch[:, 156:159].float().contiguous(),
                                                  albedo.expand(n, -1, -1, -1), lights.expand(n, -1, -1))[2]
        yy, xx = torch.meshgrid(torch.linspace(-1, 1, 256), torch.linspace(-1, 1, 256), indexing="ij")
        region = ((xx / 0.8) ** 2 + (yy / 0.9) ** 2 < 1).float()[None, None].to(device)      # stand-in for face_region_mask_file
        return InterpolatedTextureLoss(max_images_in_batch, FlameTextureSpace(synthetic_texture_data(), flame=flame), render_condition,
                                       region, rng="device")

    # ------------------------------------------------------------------------------------------- CUDA graphs
    def capture(self, batch, resolution):
        """Capture the iteration into CUDA graphs so that a step is a handful of cudaGraphLaunch calls instead of ~2000
        kernel launches issued from Python.  The iteration is cut at the two gradient exchanges, which stay OUTSIDE the
        graphs (eager ``torch.distributed`` all-reduce on the same stream):
            seg 1: generator forward, D forward x2 (+R1), D backward      | all-reduce D grads
            seg 2: D Adam step, D forward on fake, G (and PPL) backward   | all-reduce G grads
            seg 3: G Adam step, EMA
        x 2 variants (iteration with / without the R1 penalty).  Call after a few eager warm-up iterations (optimiser
        state and workspaces must exist).  ``train_iteration`` then copies its inputs into the static buffers and replays."""
        from . import _lib
        dev = self.device
        self._static = (torch.zeros(batch, 3, resolution, resolution, device=dev),
                        torch.zeros(batch, 6, resolution, resolution, device=dev),
                        torch.zeros(batch, dtype=torch.long, device=dev))
        if self.interp_tex_loss is not None:
            self._static = self._static + (torch.zeros(batch, 159, device=dev),)
        graphs, pool = {}, None
        self.graph_launches = {}
        torch.cuda.synchronize()
        for with_r1 in (True, False):
            n0 = _lib.launch_count()
            segs, state = [], {}
            for seg in (self._seg1, self._seg2, self._seg3):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, pool=pool):
                    if seg == self._seg2:
                        seg(state, *self._static[:3], with_r1, *self._static[3:])
                    else:
                        seg(state, *self._static[:3], with_r1)
                pool = g.pool()
                segs.append(g)
            self.graph_launches[with_r1] = _lib.launch_count() - n0      # gif_b200 kernel nodes per replayed iteration
            graphs[with_r1] = (segs, (state["d_loss"], state["g_loss"]))
        self._graphs = graphs
        # a replay writes the parameters without running Python, so their version counters do not move: bumped by hand
        self._replay_written = [p for m in (self.generator, self.discriminator, self.g_running) for p in m.parameters()]

    def train_iteration(self, real_image, flm_rndr, input_indices, flm_lbls=None):
        """real_image (B,3,R,R) in [-1,1], flm_rndr (B,6,R,R) in [-1,1], input_indices (B,) int64 -- device tensors (or
        pinned host tensors when CUDA graphs are active); flm_lbls (B,159) FLAME labels [shape|exp|pose|cam], needed only
        with ``texture_loss=True``.  Returns (d_loss, g_loss) as 0-d device tensors."""
        extra = () if self.interp_tex_loss is None else (flm_lbls,)
        with_r1 = (self.iteration + 1) % self.r1_every == 0                       # train.py:145
        self.iteration += 1
        if self._graphs is not None:
            self.replayed_launches = getattr(self, "replayed_launches", 0) + self.graph_launches[with_r1]
            for dst, src in zip(self._static, (real_image, flm_rndr, input_indices) + extra):
                dst.copy_(src, non_blocking=True)
            (g1, g2, g3), out = self._graphs[with_r1]
            g1.replay()
            self.d_reducer.reduce()                 # the pack (multi-tensor copy into the flat buffer) is the tail of graph 1
            g2.replay()
            self.g_reducer.reduce()
            g3.replay()
            torch.autograd.graph.increment_version(self._replay_written)
            return out
        state = {}
        self._seg1(state, real_image, flm_rndr, input_indices, with_r1)
        self.d_reducer.reduce()
        self._seg2(state, real_image, flm_rndr, input_indices, with_r1, *extra)
        self.g_reducer.reduce()
        self._seg3(state, real_image, flm_rndr, input_indices, with_r1)
        return state["d_loss"], state["g_loss"]

    def _seg1(self, st, real_image, flm_rndr, input_indices, with_r1):
        G, D, step = self.generator, self.discriminator, self.step_idx
        # ------------------------------------------------ shared generator forward (train.py:157 == train.py:197)
        requires_grad(G, True)
        w = G.z_to_w(G.img_embdng(input_indices))                                # gen.py:275
        fake = losses._synth_from_w(G, w, flm_rndr, step)                         # the graph is reused by the G step
        # ------------------------------------------------ D step (train.py:82-178)
        requires_grad(D, True)
        self.d_reducer.zero()
        real_image = real_image.detach().requires_grad_(True)                     # train.py:135-136
        real_scores, _ = D([real_image], condition=flm_rndr, step=step, alpha=1)
        real_loss = F.softplus(-real_scores).mean()
        if with_r1:                                                               # train.py:145-149
            real_loss = real_loss + losses.grad_penalty_loss([real_image], real_scores, step=None).mean()
        fake_scores, _ = D([fake.detach()], condition=flm_rndr, step=step, alpha=1)   # train.py:160-170
        d_loss = real_loss + F.softplus(fake_scores).mean()
        # 1/world folded into the backward seed: the SUM all-reduce then leaves the mean gradient (no scaling pass)
        (d_loss * self.d_reducer.pre_scale() if world_gt1(self.d_reducer) else d_loss).backward()
        self.d_reducer.pack()                      # world > 1: gradients -> flat buffer (capturable); the collective follows
        st.update(w=w, fake=fake, d_loss=d_loss.detach())

    def _seg2(self, st, real_image, flm_rndr, input_indices, with_r1, flm_lbls=None):
        G, D, step = self.generator, self.discriminator, self.step_idx
        self.d_optimizer.step()
        # ------------------------------------------------ G step (train.py:181-252)
        requires_grad(D, False)
        self.g_reducer.zero()
        predict, _ = D([st["fake"]], condition=flm_rndr, step=step, alpha=1)      # the UPDATED discriminator (train.py:200)
        g_loss = F.softplus(-predict).mean()
        if self.ppl is not None:                                                  # train.py:205-208, weight 2
            g_loss = g_loss + 2 * self.ppl.path_length_from(st["fake"], st["w"])
        if self.embedding_reg_weight != 0.0:                                      # train.py:216-219
            g_loss = g_loss + self.embedding_reg_weight * losses.l2_reg(G.z_to_w)
        if self.interp_tex_loss is not None:                                      # train.py:224-238
            u = torch.rand((), device=flm_lbls.device)                            # np.random.uniform(0, 1) there; device RNG here
            flm_intrp = flm_lbls[:-1, :159] + u * (flm_lbls[1:, :159] - flm_lbls[:-1, :159])
            interp = self.interp_tex_loss.tex_sp_intrp_loss(
                flm_intrp, G, step=step, alpha=1, max_ids=self.vocab, normal_maps_as_cond=True,
                use_posed_constant_input=False, rendered_flame_as_condition=True)
            if self.adaptive_interp_loss:                                         # train.py:236-237
                interp = interp * (0.25 * g_loss.detach() / interp.detach())
            g_loss = g_loss + interp
        (g_loss * self.g_reducer.pre_scale() if world_gt1(self.g_reducer) else g_loss).backward()
        self.g_reducer.pack()
        st["g_loss"] = g_loss.detach()
        st.pop("fake")
        st.pop("w")

    def _seg3(self, st, real_image, flm_rndr, input_indices, with_r1):
        G = self.generator
        self.g_optimizer.step()
        accumulate(self.g_running, G, decay=0.5 ** (32 / (10 * 1000)))            # train.py:250
        requires_grad(G, False)
