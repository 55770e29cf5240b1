"""Scene-completion sampling pipeline — mirror of the reference's `DiffCompletion`
(/root/reference/lidiff/tools/diff_completion_pipeline.py:15-169): same method names, argument
meaning and data flow (float64 `x_init`, float32 TensorField features, classifier-free guidance,
DPM-Solver++(2M) SDE, refinement net + 6x offsets).

Two execution paths over the same CUDA library:
  * operator path  (`engine=False`): every line of the reference loop as one operator call on the
    lidiff_b200 ME / keops / diffusers surface — what the reference's own scripts get through the shims;
  * fused engine   (`engine=True`, default): `lidiff_b200.engine.DenoiseEngine`, the sync-free
    restructured loop (SURVEY.md App. D) the benchmark measures.
Noise can be injected (`start_noise`, `step_noise`) for reproducible parity tests; by default it is
drawn with torch.randn exactly where the reference draws it.
"""
from __future__ import annotations

import copy
import gc

import numpy as np
import torch
import torch.nn as nn

from . import me as ME
from . import minkunet as minknet
from .scheduler import DPMSolverMultistepScheduler

# batches of at least this many scans sample their points with the cluster kernel (all scans at once); smaller ones with the
# single-scan kernel per scan, which is faster below that (scripts/bench_batch.py, DESIGN.md §3)
FPS_CLUSTER_MIN_SCANS = 3

DEFAULT_HPARAMS = {       # /root/reference/lidiff/config/config.yaml
    "data": {"resolution": 0.05, "num_points": 180000, "max_range": 50.0},
    "train": {"uncond_w": 6.0},
    "diff": {"beta_start": 3.5e-5, "beta_end": 0.007, "beta_func": "linear", "t_steps": 1000, "s_steps": 50},
    "model": {"out_dim": 96},
}


class DiffCompletion(nn.Module):
    def __init__(self, diff_path=None, refine_path=None, denoising_steps=50, cond_weight=6.0, *,
                 state_dicts=None, hparams=None, device="cuda", engine=True, conv_algo=0):
        super().__init__()
        hp = copy.deepcopy(DEFAULT_HPARAMS)
        ckpt_diff = ckpt_refine = None
        if diff_path is not None:
            ckpt_diff = torch.load(diff_path, map_location="cpu", weights_only=False)
            for k, v in ckpt_diff.get("hyper_parameters", {}).items():
                hp.setdefault(k, {}).update(v) if isinstance(v, dict) else hp.__setitem__(k, v)
        if hparams:
            for k, v in hparams.items():
                hp.setdefault(k, {}).update(v)
        self.hparams = hp
        assert denoising_steps <= hp["diff"]["t_steps"], \
            f"The number of denoising steps cannot be bigger than T={hp['diff']['t_steps']} (you've set '-T {denoising_steps}')"

        self.partial_enc = minknet.MinkGlobalEnc(in_channels=3, out_channels=hp["model"]["out_dim"])
        self.model = minknet.MinkUNetDiff(in_channels=3, out_channels=hp["model"]["out_dim"])
        self.model_refine = minknet.MinkUNet(in_channels=3, out_channels=3 * 6)
        if ckpt_diff is not None:
            self.load_state_dict(ckpt_diff["state_dict"], strict=False)
        if refine_path is not None:
            ckpt_refine = torch.load(refine_path, map_location="cpu", weights_only=False)
            self.load_state_dict(ckpt_refine["state_dict"], strict=False)
        if state_dicts is not None:        # {"enc":..., "diff":..., "refine":...} with the reference's key names
            self.partial_enc.load_state_dict(state_dicts["enc"])
            self.model.load_state_dict(state_dicts["diff"])
            if state_dicts.get("refine") is not None:
                self.model_refine.load_state_dict(state_dicts["refine"])
        self.eval()
        self.to(device)
        self._device = torch.device(device)
        for m in self.modules():
            if isinstance(m, (ME.MinkowskiConvolution, ME.MinkowskiConvolutionTranspose)):
                m.algo = conv_algo

        hp["diff"]["s_steps"] = denoising_steps
        self.dpm_scheduler = DPMSolverMultistepScheduler(
            num_train_timesteps=hp["diff"]["t_steps"], beta_start=hp["diff"]["beta_start"],
            beta_end=hp["diff"]["beta_end"], beta_schedule="linear", algorithm_type="sde-dpmsolver++", solver_order=2)
        self.dpm_scheduler.set_timesteps(hp["diff"]["s_steps"])
        self.scheduler_to_cuda()
        hp["train"]["uncond_w"] = cond_weight
        hp["data"]["max_range"] = 50.0
        self.w_uncond = hp["train"]["uncond_w"]
        self.use_engine = engine
        self._engine = None              # the one fused engine alive, sized for the batch size in use
        self._last_batch = 1             # batch size of the last trajectory (a different one starts fresh)

    device = property(lambda self: self._device)

    def scheduler_to_cuda(self):
        s = self.dpm_scheduler
        for name in ("timesteps", "betas", "alphas", "alphas_cumprod", "alpha_t", "sigma_t", "lambda_t", "sigmas"):
            setattr(s, name, getattr(s, name).to(self.device))

    # ---- reference: points_to_tensor :68-84 -----------------------------------------------------
    def points_to_tensor(self, points):
        x_feats = ME.utils.batched_coordinates(list(points[:]), dtype=torch.float32, device=self.device)
        x_coord = torch.round(x_feats.clone() / self.hparams["data"]["resolution"])
        return ME.TensorField(features=x_feats[:, 1:], coordinates=x_coord,
                              quantization_mode=ME.SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE,
                              minkowski_algorithm=ME.MinkowskiAlgorithm.SPEED_OPTIMIZED, device=self.device)

    def reset_partial_pcd(self, x_part, x_uncond):
        x_part = self.points_to_tensor(x_part.F.reshape(1, -1, 3).detach())
        x_uncond = self.points_to_tensor(torch.zeros_like(x_part.F.reshape(1, -1, 3)))
        return x_part, x_uncond

    # ---- reference: preprocess_scan :92-105 (range filter + FPS + x10 repeat) ---------------------
    def preprocess_scan(self, scan):
        from .preprocess import farthest_point_sample
        scan = np.asarray(scan)
        dist = np.sqrt(np.sum(scan ** 2, -1))
        scan = scan[(dist < self.hparams["data"]["max_range"]) & (dist > 3.5)][:, :3]
        pts = torch.as_tensor(scan, dtype=torch.float64, device=self.device)
        sel = farthest_point_sample(pts, int(self.hparams["data"]["num_points"] / 10))
        return pts[sel].repeat(10, 1)[None, :, :]

    def preprocess_scans(self, scans):
        """preprocess_scan of every scan, the farthest point sampling of all of them in one launch -> (B, num_points, 3) fp64"""
        from .preprocess import farthest_point_sample, farthest_point_sample_batched
        pts = []
        for scan in scans:
            scan = np.asarray(scan)
            dist = np.sqrt(np.sum(scan ** 2, -1))
            pts.append(torch.as_tensor(scan[(dist < self.hparams["data"]["max_range"]) & (dist > 3.5)][:, :3], dtype=torch.float64,
                                       device=self.device))
        n_s = int(self.hparams["data"]["num_points"] / 10)
        if len(pts) >= FPS_CLUSTER_MIN_SCANS:
            sel = farthest_point_sample_batched(pts, n_s)
        else:
            sel = [farthest_point_sample(p, n_s) for p in pts]
        return torch.stack([p[s].repeat(10, 1) for p, s in zip(pts, sel)])

    def postprocess_scan(self, completed_scan, input_scan):
        dist = np.sqrt(np.sum(completed_scan ** 2, -1))
        post_scan = completed_scan[dist < self.hparams["data"]["max_range"]]
        max_z = input_scan[..., 2].max().item()
        min_z = (input_scan[..., 2].mean() - 2 * input_scan[..., 2].std()).item()
        return post_scan[(post_scan[:, 2] < max_z) & (post_scan[:, 2] > min_z)]

    # ---- reference: complete_scan :117-132 --------------------------------------------------------
    def complete_scan(self, scan, start_noise=None, step_noise=None, preprocessed=False, fresh=False):
        """fresh=False (default) keeps the scheduler's multistep state between scans like the reference does (its main loop,
        :213-222, never calls set_timesteps again: the first update of every scan after the first is second-order against the
        previous scan's last x0); fresh=True starts a new trajectory."""
        fresh = fresh or self._last_batch != 1      # after a batch of another size the multistep state does not fit this scan
        self._last_batch = 1
        scan = scan if preprocessed else self.preprocess_scan(scan)
        scan = scan.to(self.device)
        if start_noise is None:
            start_noise = torch.randn(scan.shape, device=self.device)
        x_feats = scan + start_noise.to(self.device)
        if self.use_engine:                     # fused path: loop, postprocess, refinement forward and the 6 offsets stay on the device
            refined, post = self.engine().complete(scan, x_feats, step_noise, fresh=fresh)
            return refined.cpu().numpy(), post.cpu().numpy()
        x_full = self.points_to_tensor(x_feats)
        x_cond = self.points_to_tensor(scan)
        x_uncond = self.points_to_tensor(torch.zeros_like(scan))
        completed_scan = self.completion_loop(scan, x_full, x_cond, x_uncond, step_noise, fresh=fresh)
        post_scan = self.postprocess_scan(completed_scan, scan)
        refine_in = self.points_to_tensor(torch.as_tensor(post_scan)[None, :, :])
        offset = self.refine_forward(refine_in).reshape(-1, 6, 3)
        refine_complete_scan = post_scan[:, None, :] + offset.cpu().numpy()
        return refine_complete_scan.reshape(-1, 3), post_scan

    def complete_scans(self, scans, start_noise=None, step_noise=None, preprocessed=False, fresh=False):
        """complete_scan of B scans that share every launch: one trajectory per scan in batch column b, as the reference's
        batched p_sample_loop (lidiff/models/models.py:132-151) samples them.  start_noise (B,N,3), step_noise (T,B,N,3); by
        default the noise is drawn once per step with shape (B,N,3).  Returns [(refined, post)] per scan, each what
        complete_scan(scans[b], start_noise[b], step_noise[:, b], fresh=True) gives up to the fp32 rounding of the sparse
        convolutions, which depends on the rows that share a tile (DESIGN.md §3, batched sampling).  fresh=False carries every slot's multistep
        state into the next batch of the same size; a batch of another size (a short last batch) starts fresh."""
        B = len(scans)
        fresh = fresh or B != self._last_batch
        if B == 1:
            r = self.complete_scan(scans[0], None if start_noise is None else start_noise[0:1],
                                   None if step_noise is None else step_noise[:, 0], preprocessed=preprocessed, fresh=fresh)
            return [r]
        self._last_batch = B
        x_init = (torch.stack([torch.as_tensor(s).reshape(-1, 3) for s in scans]) if preprocessed else self.preprocess_scans(scans))
        x_init = x_init.to(self.device)
        if start_noise is None:
            start_noise = torch.randn(x_init.shape, device=self.device)
        x_feats = x_init + start_noise.to(self.device)
        if self.use_engine:
            outs = self.engine(B).complete_batch(x_init, x_feats, step_noise, fresh=fresh)
            return [(r.cpu().numpy(), p.cpu().numpy()) for r, p in outs]
        x_full = self.points_to_tensor(x_feats)
        x_cond = self.points_to_tensor(x_init)
        x_uncond = self.points_to_tensor(torch.zeros_like(x_init))
        completed = self.completion_loop_batch(x_init, x_full, x_cond, x_uncond, step_noise, fresh=fresh).reshape(B, -1, 3)
        posts = [self.postprocess_scan(completed[b], x_init[b]) for b in range(B)]
        refine_in = self.points_to_tensor([torch.as_tensor(p) for p in posts])
        offset = self.refine_forward(refine_in).reshape(-1, 6, 3).cpu().numpy()
        out, k = [], 0
        for p in posts:
            out.append(((p[:, None, :] + offset[k:k + p.shape[0]]).reshape(-1, 3), p))
            k += p.shape[0]
        return out

    def completion_loop_batch(self, x_init, x_t, x_cond, x_uncond, step_noise=None, fresh=False):
        """completion_loop over B scans in one TensorField (x_init (B,N,3)), as the reference's p_sample_loop runs it: the
        timestep repeated per scan, one scheduler step over (B,N,3)"""
        self.scheduler_to_cuda()
        if fresh:
            self.dpm_scheduler.set_timesteps(self.dpm_scheduler.num_inference_steps, device=self.device)
        B = x_init.shape[0]
        for i in range(len(self.dpm_scheduler.timesteps)):
            t = torch.ones(B, dtype=torch.long, device=self.device) * self.dpm_scheduler.timesteps[i]
            noise_t = self.classfree_forward(x_t, x_cond, x_uncond, t)
            input_noise = x_t.F.reshape(B, -1, 3) - x_init
            nz = None if step_noise is None else step_noise[i].to(self.device)
            x_t = x_init + self.dpm_scheduler.step(noise_t, t[0], input_noise, noise=nz)["prev_sample"]
            x_t = self.points_to_tensor(x_t)
            x_cond = self.points_to_tensor(x_cond.F.reshape(B, -1, 3).detach())
            x_uncond = self.points_to_tensor(torch.zeros_like(x_cond.F.reshape(B, -1, 3)))
        return x_t.F.cpu().detach().numpy()

    def refine_forward(self, x_in):
        with torch.no_grad():
            return self.model_refine(x_in)

    def forward(self, x_full, x_full_sparse, x_part, t):
        with torch.no_grad():
            part_feat = self.partial_enc(x_part)
            out = self.model(x_full, x_full_sparse, part_feat, t)
        return out.reshape(t.shape[0], -1, 3)

    def classfree_forward(self, x_t, x_cond, x_uncond, t):
        x_t_sparse = x_t.sparse()
        x_cond = self.forward(x_t, x_t_sparse, x_cond, t)
        x_uncond = self.forward(x_t, x_t_sparse, x_uncond, t)
        return x_uncond + self.w_uncond * (x_cond - x_uncond)

    # ---- reference: completion_loop :155-169 ------------------------------------------------------
    def completion_loop(self, x_init, x_t, x_cond, x_uncond, step_noise=None, n_steps=None, fresh=False):
        self.scheduler_to_cuda()
        if fresh:
            self.dpm_scheduler.set_timesteps(self.dpm_scheduler.num_inference_steps, device=self.device)
        T = len(self.dpm_scheduler.timesteps) if n_steps is None else n_steps
        for i in range(T):
            t = self.dpm_scheduler.timesteps[i][None]
            noise_t = self.classfree_forward(x_t, x_cond, x_uncond, t)
            input_noise = x_t.F.reshape(t.shape[0], -1, 3) - x_init
            nz = None if step_noise is None else step_noise[i].to(self.device)
            x_t = x_init + self.dpm_scheduler.step(noise_t, t, input_noise, noise=nz)["prev_sample"]
            x_t = self.points_to_tensor(x_t)
            x_cond, x_uncond = self.reset_partial_pcd(x_cond, x_uncond)
        return x_t.F.cpu().detach().numpy()

    # ---- fused path -----------------------------------------------------------------------------------
    def engine(self, batch=1):
        """the fused engine for batches of `batch` scans.  An engine holds its buffers and step graphs for one batch size (about
        20 GiB per 180 000-point scan), so one is alive at a time: asking for another batch size (a short last batch) releases
        the current engine and returns its memory to the device before the new one is sized."""
        if self._engine is not None and self._engine.B != batch:
            self._engine = None
            gc.collect()
            if torch.cuda.is_available():
                torch.cuda.empty_cache()
        if self._engine is None:
            from .engine import DenoiseEngine
            self._engine = DenoiseEngine.from_modules(self, **({} if batch == 1 else {"batch": batch}))
        return self._engine
