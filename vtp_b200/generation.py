"""The consumer side of the encode/decode path (SURVEY.md §8f rank 2): the H100-native counterparts of
`generation/tokenizer/vtp_tokenizer.py` (class `VTP_Tokenizer`, same constructor arguments, attributes and methods) and
of the latent-extraction loop of `generation/tools/extract_features_vtp.py` (same shard files, keys and metadata).

What changes underneath, not at the surface:
  * `decode_to_images` runs inverse-normalise · 255 · clamp · uint8 · NCHW→NHWC as ONE kernel (`vtp_image_to_u8`) and
    brings 3 bytes per pixel to the host instead of 12 (the reference copies the fp32 image, vtp_tokenizer.py:114-118);
  * `LatentShardWriter` keeps the encoder busy: latents are copied to pinned host memory on a side stream (no
    `.cpu()` stall per batch, vtp_tokenizer.py:93), and the per-channel statistics behind `latents_stats.pt` are
    accumulated on the device by a fused pass over each latent batch (`vtp_latent_stats`) instead of re-reading the
    shards afterwards.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import torch

from . import lib
from .model import VTPModel

# timm.data.constants.IMAGENET_DEFAULT_MEAN / _STD (generation/tokenizer/vtp_tokenizer.py:4,11)
IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)
NORMALIZE_HALF = {"mean": [0.5, 0.5, 0.5], "std": [0.5, 0.5, 0.5]}
NORMALIZE_IMAGENET = {"mean": list(IMAGENET_DEFAULT_MEAN), "std": list(IMAGENET_DEFAULT_STD)}


class VTP_Tokenizer:
    """generation/tokenizer/vtp_tokenizer.py:14-119.  `model=` accepts an already-built VTPModel (the reference only
    loads from `hf_model_path`)."""

    def __init__(self, hf_model_path: Optional[str] = None, img_size: int = 256, horizon_flip: float = 0.5,
                 fp16: bool = True, normalize_type: str = "imagenet", model: Optional[VTPModel] = None):
        self.img_size = img_size
        self.horizon_flip = horizon_flip
        self.fp16 = fp16
        self.normalize_type = normalize_type
        self._setup_normalization(normalize_type)
        if model is None:
            if hf_model_path is None:
                raise ValueError("hf_model_path or model is required")
            model = VTPModel.from_pretrained(hf_model_path)
        self.model = model.cuda().eval()
        config = self.model.config
        self.patch_size = config.vision_patch_size
        self.embed_dim = config.vision_feature_bottleneck
        self.downsample_ratio = self.patch_size
        self.latent_size = img_size // self.downsample_ratio
        dev = self.model.trunk.cls_token.device
        self._sub = torch.tensor(self.inv_mean, dtype=torch.float32, device=dev)
        self._div = torch.tensor(self.inv_std, dtype=torch.float32, device=dev)

    def _setup_normalization(self, normalize_type: str):
        """Same attributes as vtp_tokenizer.py:56-73 (norm_mean / norm_std and the inverse pair used by `transform_inv`):
        de-normalisation x * std + mean is kept in the `Normalize(-mean / std, 1 / std)` form the reference uses, so that
        the fused uint8 kernel reproduces its arithmetic bit for bit."""
        table = {"half": NORMALIZE_HALF, "imagenet": NORMALIZE_IMAGENET}
        if normalize_type not in table:
            raise ValueError(f"Unknown normalize_type: {normalize_type}. Use 'half' or 'imagenet'.")
        self.norm_mean, self.norm_std = list(table[normalize_type]["mean"]), list(table[normalize_type]["std"])
        pairs = list(zip(self.norm_mean, self.norm_std))
        self.inv_mean, self.inv_std = [-m / s for m, s in pairs], [1.0 / s for _, s in pairs]

    def transform_inv(self, x: torch.Tensor) -> torch.Tensor:
        """torchvision Normalize(inv_mean, inv_std) on a [B,3,H,W] tensor (plain torch; for callers that want floats)."""
        sub = torch.as_tensor(self.inv_mean, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
        div = torch.as_tensor(self.inv_std, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
        return (x - sub) / div

    def img_transform(self, p_hflip: float = 0, img_size: Optional[int] = None):
        """Host-side image loading for the extraction loop: ADM centre crop -> random horizontal flip -> float tensor ->
        normalise, i.e. what vtp_tokenizer.py:75-82 composes out of torchvision transforms, as one callable (the flip draws
        `torch.rand(1)` exactly once per image, like `RandomHorizontalFlip`, so a seeded run sees the same flips)."""
        from torchvision.transforms import functional as TF

        from .image_utils import center_crop_arr

        size = self.img_size if img_size is None else img_size
        mean, std = self.norm_mean, self.norm_std

        def load(pil_image):
            img = center_crop_arr(pil_image, size)
            if bool(torch.rand(1) < p_hflip):
                img = TF.hflip(img)
            return TF.normalize(TF.to_tensor(img), mean, std, inplace=True)

        return load

    # ------------------------------------------------------------------ encode / decode (vtp_tokenizer.py:84-119)
    def encode_images_device(self, images: torch.Tensor) -> torch.Tensor:
        """Latents [B, C, H/16, W/16] left on the device (no host synchronisation)."""
        with torch.no_grad():
            if not images.is_cuda:
                images = images.cuda(non_blocking=True)
            B, C, H, W = images.shape
            self._current_img_h, self._current_img_w = H, W
            return self.model.get_reconstruction_latents(images).detach()

    def encode_images(self, images: torch.Tensor) -> torch.Tensor:
        return self.encode_images_device(images).cpu()

    def decode_to_images_device(self, z: torch.Tensor) -> torch.Tensor:
        """uint8 NHWC [B, H, W, 3] on the device."""
        with torch.no_grad():
            if not z.is_cuda:
                z = z.cuda(non_blocking=True)
            B, C, H_latent, W_latent = z.shape
            self._current_img_h = H_latent * self.patch_size
            self._current_img_w = W_latent * self.patch_size
            decoded = self.model.get_latents_decoded_images(z)
            out = torch.empty((B, decoded.shape[2], decoded.shape[3], 3), dtype=torch.uint8, device=decoded.device)
            lib.image_to_u8(decoded, self._sub, self._div, out)
            return out

    def decode_to_images(self, z: torch.Tensor):
        return self.decode_to_images_device(z).cpu().numpy()


class LatentShardWriter:
    """The extraction loop of generation/tools/extract_features_vtp.py:70-126 without its per-batch stalls.

        w = LatentShardWriter(out_dir, rank=0, shard_size=10000)
        for x, x_flip, y in loader:
            w.add(tok.encode_images_device(x), tok.encode_images_device(x_flip), y)
        w.close()            # last partial shard + latents_stats.pt

    Shards: `latents_rank{rank:02d}_shard{n:03d}.safetensors` with tensors `latents`, `latents_flip`, `labels` and the
    reference's metadata keys.  Statistics: per-channel mean / unbiased std over every un-flipped latent element,
    accumulated in fp64 on the device (LightningDiT's ImgLatentDataset — an absent submodule, .gitmodules:1-3 —
    computes the same two tensors `[1, C, 1, 1]` from a 10 000-sample subset; restated, unpinned)."""

    def __init__(self, output_dir: str, rank: int = 0, shard_size: int = 10000, device="cuda"):
        self.dir, self.rank, self.shard_size = output_dir, rank, shard_size
        os.makedirs(output_dir, exist_ok=True)
        self.device = torch.device(device)
        self.copy_stream = torch.cuda.Stream(self.device)
        self._pending: List[tuple] = []      # (event, host latents, host flipped, labels)
        self._lat: List[torch.Tensor] = []
        self._flip: List[torch.Tensor] = []
        self._lab: List[torch.Tensor] = []
        self._count = 0
        self.saved_files = 0
        self._sum = self._sumsq = None
        self._n = 0

    def add(self, latents: torch.Tensor, latents_flip: torch.Tensor, labels: torch.Tensor):
        if self._sum is None:
            C = latents.shape[1]
            self._sum = torch.zeros(C, dtype=torch.float64, device=self.device)
            self._sumsq = torch.zeros(C, dtype=torch.float64, device=self.device)
        lat = latents.contiguous()
        lib.latent_stats(lat, self._sum, self._sumsq)
        self._n += lat.numel() // lat.shape[1]
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(ready)
            h0 = torch.empty(lat.shape, dtype=lat.dtype, pin_memory=True)
            h1 = torch.empty(latents_flip.shape, dtype=latents_flip.dtype, pin_memory=True)
            h0.copy_(lat, non_blocking=True)
            h1.copy_(latents_flip, non_blocking=True)
            lat.record_stream(self.copy_stream)
            latents_flip.record_stream(self.copy_stream)
            done = torch.cuda.Event()
            done.record(self.copy_stream)
        self._pending.append((done, h0, h1, labels.detach().cpu()))
        self._drain(block=False)

    def _drain(self, block: bool):
        while self._pending and (block or self._pending[0][0].query()):
            done, h0, h1, lab = self._pending.pop(0)
            done.synchronize()
            self._lat.append(h0), self._flip.append(h1), self._lab.append(lab)
            self._count += h0.shape[0]
            if self._count >= self.shard_size:
                self._save()

    def _save(self):
        from safetensors.torch import save_file

        if not self._lat:
            return
        d = {"latents": torch.cat(self._lat, 0).contiguous(), "latents_flip": torch.cat(self._flip, 0).contiguous(),
             "labels": torch.cat(self._lab, 0).contiguous()}
        save_file(d, os.path.join(self.dir, f"latents_rank{self.rank:02d}_shard{self.saved_files:03d}.safetensors"),
                  metadata={"total_size": f"{d['latents'].shape[0]}", "dtype": f"{d['latents'].dtype}",
                            "device": f"{d['latents'].device}"})
        self._lat, self._flip, self._lab, self._count = [], [], [], 0
        self.saved_files += 1

    def stats(self) -> Dict[str, torch.Tensor]:
        """{'mean': [1,C,1,1], 'std': [1,C,1,1]} (unbiased std) of everything added so far."""
        n = float(self._n)
        s, ss = self._sum.cpu(), self._sumsq.cpu()
        mean = s / n
        var = (ss - n * mean * mean) / max(n - 1.0, 1.0)
        return {"mean": mean.float().view(1, -1, 1, 1), "std": var.clamp_min(0).sqrt().float().view(1, -1, 1, 1)}

    def close(self, write_stats: Optional[bool] = None, process_group=None):
        """Flush the last shard and write `latents_stats.pt`.  Multi-rank extraction (one writer per rank into a shared
        directory, like extract_features_vtp.py): the fp64 partial sums Σx, Σx², n are all-reduced over the process group
        (when torch.distributed is initialised) so the statistics cover every rank's latents, and ONLY rank 0 writes the
        file — the default `write_stats=None` means "rank 0 only"."""
        self._drain(block=True)
        self._save()
        import torch.distributed as dist
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1
        if self._sum is None and multi:          # a rank without data still has to join the reduction
            raise RuntimeError("LatentShardWriter.close(): this rank added no latents; every rank must add at least one batch")
        if multi:
            n = torch.tensor([float(self._n)], dtype=torch.float64, device=self.device)
            for t in (self._sum, self._sumsq, n):
                dist.all_reduce(t, group=process_group)
            self._n = int(n.item())
        if write_stats is None:
            write_stats = self.rank == 0
        if write_stats and self._sum is not None:
            torch.save(self.stats(), os.path.join(self.dir, "latents_stats.pt"))
