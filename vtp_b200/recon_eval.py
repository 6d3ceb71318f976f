"""Reconstruction evaluation on the device (tools/test_reconstruction_hf.py of the reference).

Every batch of ImageNet-normalised images is encoded (bf16 or fp32, as the reference's autocast), decoded in fp32 and
scored without a host read: `vtp_recon_pixels` denormalises and clamps both images in one pass, writes the uint8 PNG
pixels and the LPIPS network input and the per-band squared-error sums; `vtp_recon_ssim` computes torchmetrics' SSIM
over 32x32 tiles; `LPIPSMetric` runs the reference's VGG16 LPIPS fp32-accurately (bf16x3 operands); and
`vtp_recon_finalise` writes the per-image PSNR / SSIM / LPIPS and adds the batch means to fp64 device accumulators.
From the second batch of a shape on, the whole step (copy-in, encode, decode, metrics) replays one CUDA graph.  The host
reads the accumulators once, in `result()`.

Aggregation follows the reference, quirks included: PSNR is the mean over images (inf when any image is reproduced
exactly), SSIM and LPIPS are the mean of per-batch means (a ragged last batch weighs as much as a full one); over
torch.distributed ranks each metric is the mean of the ranks' means and num_samples = images per rank * world.

    python -m vtp_b200.recon_eval --model_path DIR --data_path VAL_DIR [--lpips_vgg vgg16.pth --lpips_lin vgg.pth]
    torchrun --nproc_per_node=8 -m vtp_b200.recon_eval ... --use_ddp
"""
from __future__ import annotations

import argparse
import functools
import os
import warnings
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional

import torch

from . import lib

F32 = torch.float32
IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)
IMAGE_EXTENSIONS = {".png", ".jpg", ".jpeg", ".bmp", ".tiff"}


def png_indices(batch_idx: int, batch_size: int, world: int, rank: int, n: int, total: Optional[int]) -> List[int]:
    """File indices of a batch's n images (test_reconstruction_hf.py:404-407): batch_idx·batch_size·world +
    rank·batch_size + j, stopping at the first index >= total.

    Kept as the reference has it, quirk included: under DistributedSampler a rank's last batch can be shorter than
    batch_size, and then some indices below total are never written (world 2, batch 4, 13 images: file 11 is missing).
    Such a sharded run leaves fewer than total PNGs, so the skip-if-present check never fires for it."""
    out = []
    for j in range(n):
        i = batch_idx * batch_size * world + rank * batch_size + j
        if total is not None and i >= total:
            break
        out.append(i)
    return out


def count_images_in_directory(directory: str) -> int:
    """test_reconstruction_hf.py:179-184."""
    if not os.path.exists(directory):
        return 0
    return sum(1 for f in os.listdir(directory) if os.path.splitext(f)[1].lower() in IMAGE_EXTENSIONS)


def rank_mean(values_mean: Optional[float], world: int, device) -> Optional[float]:
    """test_reconstruction_hf.py:417-422: the mean over ranks of each rank's mean (world 1: the value itself)."""
    if values_mean is None or world == 1:
        return values_mean
    import torch.distributed as dist

    t = torch.tensor(values_mean, dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t / world)


class _Step:
    """Device buffers of one batch shape (the graph's static inputs and outputs)."""

    def __init__(self, B: int, H: int, W: int, dev, lpips: bool, save: bool, fid: bool = False):
        self.x = torch.empty((B, 3, H, W), dtype=F32, device=dev)
        self.nbands = min(H, 16)
        self.sse = torch.empty((B, self.nbands), dtype=torch.float64, device=dev)
        self.ssim_part = torch.empty((B, lib.recon_ssim_tiles(H, W)), dtype=torch.float64, device=dev)
        self.psnr = torch.empty(B, dtype=torch.float64, device=dev)
        self.ssim = torch.empty(B, dtype=F32, device=dev)
        self.lpips = torch.empty(B, dtype=F32, device=dev) if lpips else None
        self.lp = torch.empty((B, 2, 3, H, W), dtype=F32, device=dev) if lpips else None
        self.u8 = torch.empty((2, B, H, W, 3), dtype=torch.uint8, device=dev) if save else None
        self.fid_rows = torch.zeros(1, dtype=torch.int32, device=dev) if fid else None  # images of the batch with a PNG
        self.graph = None
        self.seen = 0
        self.copied = None   # event: the last PNG copy out of u8 has finished


class ReconstructionEvaluator:
    """PSNR / SSIM / LPIPS of encode→decode round trips, accumulated on the device.

    model: a VTPModel on the GPU.  lpips: an `LPIPSMetric` or None (LPIPS is then reported as None).  precision: "bf16"
    or "fp32" for the encoder (the decoder always runs in fp32, as the reference).  save_dir: if given, the uint8
    reference / reconstruction images are written to save_dir/reference/ref_{i:06d}.png and save_dir/reconstructed/
    rec_{i:06d}.png by a pool of PNG writers fed through pinned buffers on a side stream.  batch_size / world / rank /
    total define the file index as the reference's DistributedSampler loop does (batch_size defaults to the first
    batch's size, total to no limit).  fid: an `FIDInception` or None; with it and save_dir, the uint8 reference and
    reconstruction images that get a PNG also go through the FID network inside the same step (rFID, see vtp_b200/fid.py),
    so the statistics cover exactly the images the PNG directories hold."""

    def __init__(self, model, lpips=None, precision: str = "bf16", save_dir: Optional[str] = None,
                 batch_size: Optional[int] = None, world: Optional[int] = None, rank: Optional[int] = None,
                 total: Optional[int] = None, use_graph: bool = True, writers: int = 4, fid=None):
        import torch.distributed as dist

        if precision not in ("bf16", "fp32"):
            raise NotImplementedError(f"precision {precision!r}: the encoder runs in 'bf16' or 'fp32' (no fp16 path)")
        self.dist = dist.is_available() and dist.is_initialized()
        self.world = int(world) if world is not None else (dist.get_world_size() if self.dist else 1)
        self.rank = int(rank) if rank is not None else (dist.get_rank() if self.dist else 0)
        self.model, self.lpips, self.precision, self.use_graph = model, lpips, precision, use_graph
        self.device = model.trunk.cls_token.device
        if self.device.type != "cuda":
            raise lib.VtpError("ReconstructionEvaluator needs the model on the CUDA device (there is no CPU path)")
        dev = self.device
        inv_mean = [-m / s for m, s in zip(IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD)]
        inv_std = [1.0 / s for s in IMAGENET_DEFAULT_STD]
        self.sub = torch.tensor(inv_mean, dtype=F32, device=dev)   # torchvision Normalize's fp32 mean / std tensors
        self.div = torch.tensor(inv_std, dtype=F32, device=dev)
        self.acc = torch.zeros(8, dtype=torch.float64, device=dev)
        self.batch_size, self.total = batch_size, total
        self.save_dir = save_dir
        self.fid = fid if save_dir is not None else None
        if self.fid is not None:
            from .fid import FIDStatistics

            self.fid_stats = (FIDStatistics(dev), FIDStatistics(dev))   # reference, reconstruction
        self._steps: Dict[tuple, _Step] = {}
        self._psnr: List[torch.Tensor] = []
        self._ssim: List[torch.Tensor] = []
        self._lpips: List[torch.Tensor] = []
        self.batches = 0
        self._pool = None
        self._pending: list = []
        self._writers = max(1, int(writers))
        if save_dir is not None:
            self.ref_dir = os.path.join(save_dir, "reference")
            self.rec_dir = os.path.join(save_dir, "reconstructed")
            os.makedirs(self.ref_dir, exist_ok=True)
            os.makedirs(self.rec_dir, exist_ok=True)
            self._pool = ThreadPoolExecutor(max_workers=self._writers)
            self._copy_stream = torch.cuda.Stream(device=dev)

    # ------------------------------------------------------------------ the device step
    def _run(self, st: _Step) -> None:
        m = self.model
        saved = m.compute_mode
        try:
            m.compute_mode = self.precision
            lat = m.get_reconstruction_latents(st.x)
            m.compute_mode = "fp32"
            rec = m.get_latents_decoded_images(lat)
        finally:
            m.compute_mode = saved
        rec = rec.contiguous()
        u8r, u8o = (st.u8[0], st.u8[1]) if st.u8 is not None else (None, None)
        lib.recon_pixels(st.x, rec, self.sub, self.div, st.sse, u8_ref=u8r, u8_rec=u8o, lp=st.lp)
        lib.recon_ssim(st.x, rec, self.sub, self.div, st.ssim_part)
        lp_part = self.lpips.parts(st.lp) if self.lpips is not None else None
        H, W = st.x.shape[-2:]
        lib.recon_finalise(st.sse, st.ssim_part, lp_part, H, W, st.psnr, st.ssim, st.lpips, self.acc)
        if self.fid is not None:
            self.fid.accumulate(st.u8[0], self.fid_stats[0], st.fid_rows)
            self.fid.accumulate(st.u8[1], self.fid_stats[1], st.fid_rows)

    @torch.no_grad()
    def add(self, images: torch.Tensor) -> None:
        """Score one batch of ImageNet-normalised fp32 images [B,3,H,W] (host, pinned or device).  Enqueues only."""
        if images.dim() != 4 or images.shape[1] != 3 or images.dtype != F32:
            raise ValueError(f"add: ImageNet-normalised fp32 [B,3,H,W] images expected, got {images.dtype} "
                             f"{tuple(images.shape)}")
        B, _, H, W = images.shape
        if H < 11 or W < 11:
            raise ValueError(f"add: SSIM's 11x11 window needs H, W >= 11, got {H}x{W}")
        if self.lpips is not None:
            self.lpips.check_shape(H, W)
        if self.batch_size is None:
            self.batch_size = B
        key = (B, H, W)
        st = self._steps.get(key)
        if st is None:
            st = self._steps[key] = _Step(B, H, W, self.device, self.lpips is not None, self.save_dir is not None,
                                          self.fid is not None)
        if st.copied is not None:
            torch.cuda.current_stream(self.device).wait_event(st.copied)  # the last batch's PNG copy has left st.u8
        st.x.copy_(images, non_blocking=True)
        idx = png_indices(self.batches, self.batch_size, self.world, self.rank, B, self.total) if self.save_dir else []
        if st.fid_rows is not None:
            st.fid_rows.fill_(len(idx))
        if self.use_graph and st.graph is None and st.seen >= 1:
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._run(st)
            st.graph = g
        if st.graph is not None:
            st.graph.replay()
        else:
            self._run(st)
        st.seen += 1
        self._psnr.append(st.psnr.clone())
        self._ssim.append(st.ssim.clone())
        if st.lpips is not None:
            self._lpips.append(st.lpips.clone())
        if self.save_dir is not None:
            self._save(st, idx)
        self.batches += 1

    def _save(self, st: _Step, idx: List[int]) -> None:
        if not idx:
            return
        n = len(idx)
        host = torch.empty((2, n) + tuple(st.u8.shape[2:]), dtype=torch.uint8, pin_memory=True)
        cs = self._copy_stream
        cs.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(cs):
            host.copy_(st.u8[:, :n], non_blocking=True)
            done = torch.cuda.Event()
            done.record(cs)
        st.copied = done
        while len(self._pending) >= 2 * self._writers:
            self._pending.pop(0).result()
        self._pending.append(self._pool.submit(_write_pngs, done, host, idx, self.ref_dir, self.rec_dir))

    # ------------------------------------------------------------------ results
    def per_image(self) -> Dict[str, torch.Tensor]:
        """Device tensors psnr [N], ssim [N] and, with LPIPS, lpips [N] of every image added so far (this rank)."""
        out = {"psnr": torch.cat(self._psnr) if self._psnr else torch.empty(0, device=self.device),
               "ssim": torch.cat(self._ssim) if self._ssim else torch.empty(0, device=self.device)}
        if self.lpips is not None:
            out["lpips"] = torch.cat(self._lpips) if self._lpips else torch.empty(0, device=self.device)
        return out

    def result(self) -> Dict[str, object]:
        """{'fid', 'psnr', 'lpips', 'ssim', 'num_samples'} aggregated as test_reconstruction_hf.py:415-466.  'fid' is None
        without an FID network (the command-line tool then computes rFID from the saved PNGs); with one, the ranks' S1,
        S2 and n are summed and rank 0 gets the Fréchet distance (the other ranks None).  Waits for the device and the
        PNG writers."""
        self.flush()
        fid = None
        if self.fid is not None:
            from .fid import frechet_distance

            if self.dist and self.world > 1:
                for s in self.fid_stats:
                    s.all_reduce()
            if self.rank == 0 and self.fid_stats[0].count() >= 2:   # a covariance needs two images
                fid = frechet_distance(*self.fid_stats[0].mu_sigma(), *self.fid_stats[1].mu_sigma())
        a = self.acc.cpu().tolist()
        n_img, n_batch = int(a[1]), int(a[4])
        psnr = a[0] / n_img if n_img else None
        ssim = a[2] / n_batch if n_batch else None
        lp = a[3] / n_batch if (n_batch and self.lpips is not None) else None
        return {"fid": fid, "psnr": rank_mean(psnr, self.world, self.device), "lpips": rank_mean(lp, self.world, self.device),
                "ssim": rank_mean(ssim, self.world, self.device), "num_samples": n_img * self.world}

    def flush(self) -> None:
        """Wait until every PNG is written (errors of a writer are raised here)."""
        while self._pending:
            self._pending.pop(0).result()

    def close(self) -> None:
        self.flush()
        if self._pool is not None:
            self._pool.shutdown(wait=True)
            self._pool = None
        for st in self._steps.values():
            if st.graph is not None:
                torch.cuda.synchronize(self.device)
                st.graph.reset()
                st.graph = None


def _write_pngs(done, host, idx, ref_dir, rec_dir) -> None:
    from PIL import Image

    done.synchronize()
    arr = host.numpy()
    for j, i in enumerate(idx):
        Image.fromarray(arr[0, j]).save(os.path.join(ref_dir, f"ref_{i:06d}.png"))
        Image.fromarray(arr[1, j]).save(os.path.join(rec_dir, f"rec_{i:06d}.png"))


# ---------------------------------------------------------------------------------------------------------- CLI
def build_parser() -> argparse.ArgumentParser:
    """The reference's flags (test_reconstruction_hf.py:471-494) plus --lpips_vgg / --lpips_lin for the LPIPS weights,
    which the reference downloads at run time."""
    ap = argparse.ArgumentParser(description="Reconstruction evaluation of a VTP checkpoint on the H100 path")
    ap.add_argument("--model_path", type=str, required=True, help="VTP checkpoint directory (config.json + safetensors)")
    ap.add_argument("--data_path", type=str, required=True, help="ImageFolder root of the evaluation images")
    ap.add_argument("--output_path", type=str, default="reconstruction_output", help="directory for the saved PNGs")
    ap.add_argument("--batch_size", type=int, default=32, help="batch size per GPU")
    ap.add_argument("--num_workers", type=int, default=4)
    ap.add_argument("--device", type=str, default="cuda:0", help="device (ignored with --use_ddp)")
    ap.add_argument("--precision", type=str, default="bf16", choices=["fp32", "fp16", "bf16"])
    ap.add_argument("--no_save_images", action="store_true", help="do not save PNGs (and skip rFID)")
    ap.add_argument("--use_ddp", action="store_true", help="data parallel over the ranks started by torchrun")
    ap.add_argument("--local_rank", type=int, default=None)
    ap.add_argument("--max_samples", type=int, default=None, help="evaluate only the first N images")
    ap.add_argument("--lpips_vgg", type=str, default=None, help="torchvision VGG16 checkpoint (features.* keys)")
    ap.add_argument("--lpips_lin", type=str, default=None, help="LPIPS lin weights (lin{0..4}.model.1.weight)")
    ap.add_argument("--fid_weights", type=str, default=None,
                    help="pytorch-fid's Inception weights (pt_inception-2015-12-05-6726825d.pth): rFID on the device")
    return ap


def make_transform(image_size: int):
    """test_reconstruction_hf.py:260-264."""
    from torchvision import transforms as Tv

    from .image_utils import center_crop_arr

    return Tv.Compose([Tv.Lambda(functools.partial(center_crop_arr, image_size=image_size)), Tv.ToTensor(),
                       Tv.Normalize(mean=IMAGENET_DEFAULT_MEAN, std=IMAGENET_DEFAULT_STD)])


def compute_fid(ref_dir: str, rec_dir: str, device) -> Optional[float]:
    """test_reconstruction_hf.py:98-104 when pytorch_fid is importable; None otherwise (this project does not build
    InceptionV3)."""
    try:
        from pytorch_fid import fid_score
    except ImportError:
        return None
    try:   # as the reference (:310-313, :435-439): a failed rFID (e.g. Inception weights not cached) is reported, not fatal
        return fid_score.calculate_fid_given_paths([ref_dir, rec_dir], batch_size=50, device=device, dims=2048,
                                                   num_workers=4)
    except Exception as e:  # noqa: BLE001 — whatever pytorch_fid raises, the other metrics are still returned
        warnings.warn(f"rFID calculation failed: {e}")
        return None


def run(args) -> Dict[str, object]:
    import torch.distributed as dist
    from torch.utils.data import DataLoader, DistributedSampler, Subset
    from torchvision.datasets import ImageFolder

    from .lpips import LPIPSMetric
    from .model import VTPModel

    if args.precision == "fp16":
        raise NotImplementedError("--precision fp16: the encoder runs in bf16 or fp32 only")
    if args.use_ddp:
        if not dist.is_initialized():
            dist.init_process_group(backend="nccl")
        local = args.local_rank if args.local_rank is not None else int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local % torch.cuda.device_count())
        device = torch.device("cuda", local % torch.cuda.device_count())
        rank, world = dist.get_rank(), dist.get_world_size()
    else:
        device, rank, world = torch.device(args.device), 0, 1
    main = rank == 0
    save = not args.no_save_images
    model = VTPModel.from_pretrained(args.model_path).to(device).eval()
    size = model.config.image_size
    use_lpips = bool(args.lpips_vgg and args.lpips_lin)
    if use_lpips:
        try:
            LPIPSMetric.check_shape(size, size)
        except ValueError as e:
            use_lpips = False
            if main:
                warnings.warn(f"{e}: LPIPS will not be calculated")
    elif main:
        warnings.warn("--lpips_vgg / --lpips_lin not given: LPIPS will not be calculated")
    dataset = ImageFolder(root=args.data_path, transform=make_transform(size))
    total = len(dataset)
    if args.max_samples is not None and args.max_samples < total:
        dataset, total = Subset(dataset, range(args.max_samples)), args.max_samples
    save_dir = os.path.join(args.output_path, "reconstructed")
    ref_dir = os.path.join(args.output_path, "reference")
    skip = bool(save and main and count_images_in_directory(save_dir) >= total and count_images_in_directory(ref_dir) >= total)
    if args.use_ddp:
        t = torch.tensor([int(skip)], device=device)
        dist.broadcast(t, src=0)
        skip = bool(t.item())
    fid_net = None
    if save and args.fid_weights:
        from .fid import FIDInception

        fid_net = FIDInception.from_file(args.fid_weights, device=device)
    if skip:
        if fid_net is not None:
            from .fid import fid_from_paths

            fid = fid_from_paths([ref_dir, save_dir], batch_size=50, num_workers=4, model=fid_net) if main else None
        else:
            fid = compute_fid(ref_dir, save_dir, device) if main else None
        if main:
            print(f"Found {total} reconstructed and reference images; skipped generation. rFID: {fid}")
        if args.use_ddp:
            dist.destroy_process_group()
        return {"fid": fid, "psnr": None, "lpips": None, "ssim": None, "num_samples": total}
    sampler = DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=False) if args.use_ddp else None
    loader = DataLoader(dataset, batch_size=args.batch_size, shuffle=False, sampler=sampler, num_workers=args.num_workers,
                        pin_memory=True)
    lpips = LPIPSMetric.from_files(args.lpips_vgg, args.lpips_lin, device=device) if use_lpips else None
    ev = ReconstructionEvaluator(model, lpips=lpips, precision=args.precision, save_dir=args.output_path if save else None,
                                 batch_size=args.batch_size, world=world, rank=rank, total=total, fid=fid_net)
    for images, _ in loader:
        ev.add(images.to(device, non_blocking=True))
    res = ev.result()
    ev.close()
    if args.use_ddp:
        dist.barrier()
    if save and main and fid_net is None:
        res["fid"] = compute_fid(ref_dir, save_dir, device)
    if main:
        print("Results:")
        if res["fid"] is not None:
            print(f"  rFID: {res['fid']:.3f}")
        if res["psnr"] is not None:
            print(f"  PSNR: {res['psnr']:.2f} dB")
        if res["lpips"] is not None:
            print(f"  LPIPS: {res['lpips']:.4f}")
        if res["ssim"] is not None:
            print(f"  SSIM: {res['ssim']:.4f}")
        print(f"  Samples: {res['num_samples']}")
    if args.use_ddp:
        dist.destroy_process_group()
    return res


def main(argv=None):
    return run(build_parser().parse_args(argv))


if __name__ == "__main__":
    main()
