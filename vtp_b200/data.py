"""Input side of the training step on the GPU / off the critical path (SURVEY.md §8f rank 4, §8 a21 "multi-crop + mask
generation").  The reference releases no training data loader (README.md:245 points at DINOv2 / OpenCLIP); what the step
consumes is fixed by `vtp/models/vtp.py:365-386,410-484`: 2 global crops (view-major) + n local crops (crop-major) per
image, iBOT `mask_indices_list` / per-patch weights over the global crops, one CLIP view + caption ids, one reconstruction
view.  A CPU loader producing that is ~1 GB of fp32 per 256-image step through PCIe plus PIL work per crop; here the
decoded uint8 images (50 MB) cross PCIe once and ONE kernel (`csrc/data.cu`) cuts, resamples, flips and normalises every
crop on the device; masks are drawn on the device; caption tokenisation (pure-Python BPE upstream,
`vtp/tokenizers/text_tokenizer.py:208-257`) runs in a worker thread under the previous step.

Crop geometry = torchvision `RandomResizedCrop.get_params` (area scale x log-uniform aspect ratio, 10 tries, centre-crop
fallback) with DINOv2's scales (global 0.32-1, local 0.05-0.32) and OpenCLIP's (0.9-1) for the contrastive view.

Photometric augmentations (`TrainBatchPipeline(photometric=PhotometricAug())`, off by default) follow DINOv2's multi-crop
recipe on the self-distillation crops only: colour jitter (p 0.8; brightness / contrast 0.4, saturation 0.2, hue 0.1, random
order), grayscale (p 0.2), Gaussian blur (9 taps, sigma U[0.1, 2]; p 1.0 / 0.1 / 0.5 on global view 1 / global view 2 /
local crops), solarise (p 0.2, global view 2 only).  The host draws one 8-float row per crop (`photometric_params`) and
`csrc/data.cu` applies them in the same pass that cuts the crop, with torchvision.transforms.v2.functional's float-image
semantics.  Deliberate differences from DINOv2's PIL pipeline: the resample is bilinear (DINOv2: bicubic) and every stage
stays fp32 (PIL rounds to uint8 after each op).  The CLIP and reconstruction views are never augmented.

Masks: exactly round(mask_ratio * HW) patches on exactly round(mask_prob * 2B) global crops (SURVEY.md §8d), static shapes so that the step stays CUDA-graph replayable."""
from __future__ import annotations

import math
from concurrent.futures import Future, ThreadPoolExecutor
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib

IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
CLIP_MEAN, CLIP_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)


def random_resized_crop_boxes(rng: np.random.Generator, n: int, H: int, W: int, scale: Tuple[float, float],
                              ratio: Tuple[float, float] = (3 / 4, 4 / 3)) -> np.ndarray:
    """torchvision.transforms.RandomResizedCrop.get_params, vectorised: n boxes (x0, y0, w, h) in source pixels."""
    area = H * W
    out = np.zeros((n, 4), dtype=np.float32)
    done = np.zeros(n, dtype=bool)
    log_r = (math.log(ratio[0]), math.log(ratio[1]))
    for _ in range(10):
        ta = area * rng.uniform(scale[0], scale[1], n)
        ar = np.exp(rng.uniform(log_r[0], log_r[1], n))
        w = np.round(np.sqrt(ta * ar)).astype(np.int64)
        h = np.round(np.sqrt(ta / ar)).astype(np.int64)
        ok = (~done) & (w > 0) & (w <= W) & (h > 0) & (h <= H)
        y0 = (rng.random(n) * (H - h + 1)).astype(np.int64)
        x0 = (rng.random(n) * (W - w + 1)).astype(np.int64)
        out[ok] = np.stack([x0, y0, w, h], 1)[ok]
        done |= ok
    if not done.all():  # fallback: central crop clipped to the ratio range
        in_r = W / H
        if in_r < ratio[0]:
            w, h = W, int(round(W / ratio[0]))
        elif in_r > ratio[1]:
            h, w = H, int(round(H * ratio[1]))
        else:
            w, h = W, H
        out[~done] = np.array([(W - w) // 2, (H - h) // 2, w, h], dtype=np.float32)
    return out


@dataclass(frozen=True)
class PhotometricAug:
    """DINO / DINOv2 photometric recipe for the self-distillation crops (defaults = the published values)."""
    jitter_p: float = 0.8
    brightness: float = 0.4          # factor U[1 - b, 1 + b]
    contrast: float = 0.4            # factor U[1 - c, 1 + c]
    saturation: float = 0.2          # factor U[1 - s, 1 + s]
    hue: float = 0.1                 # shift U[-h, h]
    gray_p: float = 0.2
    blur_sigma: Tuple[float, float] = (0.1, 2.0)
    blur_p: Tuple[float, float, float] = (1.0, 0.1, 0.5)   # global view 1, global view 2, local crops
    solarize_p: float = 0.2          # global view 2 only
    solarize_threshold: float = 128 / 255


PHOTO_OFF = (0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 2.0)   # a params row with every stage off


def photometric_params(rng: np.random.Generator, n: int, aug: PhotometricAug, blur_p: float, solarize_p: float) -> np.ndarray:
    """n rows of the vtp_crop_augment table (fp32 [n, 8], layout in include/vtp_b200.h): jitter factors and a uniform
    order code 0..23 into itertools.permutations(range(4)) (-1 = no jitter), grayscale flag, blur sigma (0 = off),
    solarise threshold (2.0 = off)."""
    out = np.empty((n, 8), dtype=np.float32)
    jit = rng.random(n) < aug.jitter_p
    out[:, 0] = rng.uniform(1 - aug.brightness, 1 + aug.brightness, n)
    out[:, 1] = rng.uniform(1 - aug.contrast, 1 + aug.contrast, n)
    out[:, 2] = rng.uniform(1 - aug.saturation, 1 + aug.saturation, n)
    out[:, 3] = rng.uniform(-aug.hue, aug.hue, n)
    out[:, 4] = np.where(jit, rng.integers(0, 24, n), -1)
    out[:, 5] = rng.random(n) < aug.gray_p
    sigma = rng.uniform(aug.blur_sigma[0], aug.blur_sigma[1], n)
    out[:, 6] = np.where(rng.random(n) < blur_p, sigma, 0.0)
    out[:, 7] = np.where(rng.random(n) < solarize_p, aug.solarize_threshold, 2.0)
    return out


def ibot_masks(n_images: int, HW: int, mask_ratio: float, mask_prob: float, device, generator: Optional[torch.Generator] = None):
    """Device-side iBOT masks of fixed size: (mask_indices int64 ascending flat indices into [n_images*HW],
    masks_weight fp32 = 1 / #masked patches of that image) — `mask_indices_list` / `masks_weight` of vtp.py:434,472."""
    n_sel = max(1, int(round(mask_prob * n_images)))
    n_mask = max(1, int(round(mask_ratio * HW)))
    sel = torch.randperm(n_images, device=device, generator=generator)[:n_sel].sort().values
    pick = torch.rand(n_sel, HW, device=device, generator=generator).topk(n_mask, dim=1).indices.sort(dim=1).values
    idx = (sel[:, None] * HW + pick).reshape(-1)
    return idx, torch.full((n_sel * n_mask,), 1.0 / n_mask, dtype=torch.float32, device=device)


class TrainBatchPipeline:
    """uint8 source images (+ captions) -> the device batch dict of `VTPTrainer.train_step`, one step ahead.

        from vtp_b200.text_tokenizer import get_tokenizer              # the reference's BPE, same ids (or any callable
        pipe = TrainBatchPipeline("cuda", tokenizer=get_tokenizer())      #   list[str] -> int64 [B, 77])
        pipe.submit(images_u8, captions)            # images: uint8 [B, H, W, 3] (pinned host or device)
        for ...:
            batch = pipe.get(); pipe.submit(next_images, next_captions)   # prepared under the step that follows
            trainer.train_step(batch)               # or replay_step(batch)

    `state_dict()` / `load_state_dict()` carry the RNG streams over a restart (`VTPTrainer.save_checkpoint(path,
    pipeline=pipe)` stores them): the resumed pipeline, given the images of the batches that were still queued, prepares
    them bit for bit as this one did.
    """

    def __init__(self, device="cuda", *, image_size: int = 256, local_size: int = 96, n_local: int = 8, patch: int = 16,
                 global_scale=(0.32, 1.0), local_scale=(0.05, 0.32), clip_scale=(0.9, 1.0), mask_ratio: float = 0.3,
                 mask_prob: float = 0.5, tokenizer: Optional[Callable[[Sequence[str]], torch.Tensor]] = None, seed: int = 0,
                 clip_norm=(CLIP_MEAN, CLIP_STD), image_norm=(IMAGENET_MEAN, IMAGENET_STD),
                 photometric: Optional[PhotometricAug] = None):
        self.device = torch.device(device)
        self.S, self.Sl, self.n_local, self.patch = image_size, local_size, n_local, patch
        self.scales = dict(g=global_scale, l=local_scale, c=clip_scale)
        self.mask_ratio, self.mask_prob = mask_ratio, mask_prob
        self.tokenizer = tokenizer
        self.rng = np.random.default_rng(seed)
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(seed)
        self.clip_norm, self.image_norm = clip_norm, image_norm
        # photometric rows come from their own generator, so boxes, flips and masks do not depend on `photometric`;
        # per step: global view 1 (B rows), global view 2 (B rows), local crops (n_local * B rows), in that order
        self.photometric = photometric
        self.photo_rng = np.random.default_rng([seed, 1])
        self._mean_ws: Dict[int, torch.Tensor] = {}
        self.stream = torch.cuda.Stream(self.device)
        self.pool = ThreadPoolExecutor(max_workers=1)
        # (batch, ready event, caption future, RNG state before the batch's draws)
        self._queue: List[Tuple[Dict[str, torch.Tensor], torch.cuda.Event, Optional[Future], dict]] = []

    def _rng_state(self) -> dict:
        return {"rng": self.rng.bit_generator.state, "photo_rng": self.photo_rng.bit_generator.state,
                "gen": bytes(self.gen.get_state().numpy())}

    def state_dict(self) -> dict:
        """The RNG streams (boxes and flips, photometric rows, iBOT masks) as they were before the oldest batch not yet
        returned by get(), or as they are now when none is queued: a pipeline that loads this state and is given the
        images of the batches still queued here, in order, prepares them bit for bit as this one does.  The NumPy states
        are JSON-serialisable dicts, the CUDA generator's state is bytes."""
        return self._queue[0][3] if self._queue else self._rng_state()

    def check_loadable(self) -> None:
        if self._queue:
            raise ValueError(f"load_state_dict() with {len(self._queue)} batch(es) queued: they were drawn from the "
                             f"current streams; get() them first")

    def load_state_dict(self, state: dict) -> None:
        """Restore state_dict()'s RNG streams; the next submit() draws what the saving pipeline drew for its batch."""
        self.check_loadable()
        self.rng.bit_generator.state = state["rng"]
        self.photo_rng.bit_generator.state = state["photo_rng"]
        self.gen.set_state(torch.frombuffer(bytearray(state["gen"]), dtype=torch.uint8))

    def _crops(self, src: torch.Tensor, n_per: int, size: int, scale, norm, flip: bool = True,
               photo: Optional[np.ndarray] = None) -> torch.Tensor:
        """n_per crops per source image, crop-major [n_per * B] (crop j of image b at row j * B + b); `photo`: one
        vtp_crop_augment row per crop, or None for plain crops."""
        B, H, W, _ = src.shape
        N = n_per * B
        boxes = random_resized_crop_boxes(self.rng, N, H, W, scale)
        idx = np.tile(np.arange(B, dtype=np.int32), n_per)
        flips = (self.rng.random(N) < 0.5).astype(np.uint8) if flip else np.zeros(N, np.uint8)
        dev = self.device
        bx = torch.from_numpy(boxes).pin_memory().to(dev, non_blocking=True)
        ix = torch.from_numpy(idx).pin_memory().to(dev, non_blocking=True)
        fl = torch.from_numpy(flips).pin_memory().to(dev, non_blocking=True)
        out = torch.empty((N, 3, size, size), dtype=torch.float32, device=dev)
        if photo is None:
            lib.crop_resize_norm(src, ix, bx, fl, out, mean=norm[0], std=norm[1])
            return out
        prm = torch.from_numpy(photo).pin_memory().to(dev, non_blocking=True)
        if N not in self._mean_ws:
            self._mean_ws[N] = torch.empty(N, dtype=torch.float32, device=dev)
        lib.crop_augment(src, ix, bx, fl, prm, self._mean_ws[N], out, mean=norm[0], std=norm[1])
        return out

    def submit(self, images_u8: torch.Tensor, captions=None) -> None:
        """images_u8: uint8 [B, H, W, 3]; captions: list[str] (needs `tokenizer`) or int64 ids [B, L] or None."""
        assert images_u8.dtype == torch.uint8 and images_u8.dim() == 4 and images_u8.shape[-1] == 3
        state = self._rng_state()
        fut = None
        ids = None
        if captions is not None and not torch.is_tensor(captions):
            if self.tokenizer is None:
                raise ValueError("captions given as strings but no tokenizer was supplied")
            fut = self.pool.submit(lambda c=list(captions): self.tokenizer(c).to(torch.long).contiguous().pin_memory())
        elif captions is not None:
            ids = captions.to(torch.long).contiguous()
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            src = images_u8.to(self.device, non_blocking=True).contiguous()
            B = src.shape[0]
            HW = (self.S // self.patch) ** 2
            pg = pl = None
            if self.photometric is not None:
                a, r = self.photometric, self.photo_rng
                pg = np.concatenate([photometric_params(r, B, a, a.blur_p[0], 0.0),
                                     photometric_params(r, B, a, a.blur_p[1], a.solarize_p)])
                pl = photometric_params(r, self.n_local * B, a, a.blur_p[2], 0.0)
            batch = dict(
                image=self._crops(src, 1, self.S, self.scales["c"], self.clip_norm, flip=False),
                global_crops=self._crops(src, 2, self.S, self.scales["g"], self.image_norm, photo=pg),  # view-major [2B]
                local_crops=self._crops(src, self.n_local, self.Sl, self.scales["l"], self.image_norm, photo=pl),
                rec_image=self._crops(src, 1, self.S, (1.0, 1.0), self.image_norm, flip=False),
            )
            batch["mask_indices"], batch["masks_weight"] = ibot_masks(2 * B, HW, self.mask_ratio, self.mask_prob, self.device, self.gen)
            if ids is not None:
                batch["text"] = ids.to(self.device, non_blocking=True)
            src.record_stream(self.stream)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._queue.append((batch, ev, fut, state))

    def get(self) -> Dict[str, torch.Tensor]:
        batch, ev, fut, _ = self._queue.pop(0)
        if fut is not None:
            batch["text"] = fut.result().to(self.device, non_blocking=True)
        torch.cuda.current_stream(self.device).wait_event(ev)
        return batch

    def close(self):
        self.pool.shutdown(wait=True)
