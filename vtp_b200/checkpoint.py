"""The on-disk format of a training checkpoint: a directory that `VTPTrainer.save_checkpoint` writes and
`VTPTrainer.load_checkpoint` reads.  This module is the only place that knows the layout; no pickle is involved.

    <path>/trainer.safetensors      fp32 state of the step, identical on every rank (written by rank 0)
    <path>/rng_rank{r:02d}.safetensors
                                    rank r's CUDA generator state (uint8) and, when given, its input pipeline's RNG state
                                    (JSON metadata for the NumPy streams, uint8 tensors for the byte-valued entries)
    <path>/checkpoint.json          the manifest: format version, step, world size, configs, every file with its byte size

A save writes into `<path>.tmp`, fsyncs every file, waits for every rank and then renames the directory into place, with
the manifest written last: an interrupted save leaves at most a `.tmp` directory, never something that reads as a
checkpoint.  A load checks the manifest, the file sizes and every tensor name, shape and dtype against what the caller
expects before it hands anything out, so a mismatched checkpoint is refused before the trainer is touched.
"""
from __future__ import annotations

import json
import os
import shutil
import struct
from typing import Dict, Iterable, List, Mapping, Optional, Sequence, Tuple

import torch

FORMAT = "vtp-train-checkpoint"
VERSION = 1
MANIFEST = "checkpoint.json"
STATE_FILE = "trainer.safetensors"

_DTYPES = {torch.float32: "F32", torch.uint8: "U8"}


def rng_file(rank: int) -> str:
    return f"rng_rank{rank:02d}.safetensors"


def state_spec(entries: Iterable, center_dim: int) -> Dict[str, Tuple[int, ...]]:
    """Name -> shape of every fp32 tensor in `trainer.safetensors` for the parameter-table `entries` (params.Entry):
    master weights, both Adam moments and the EMA teacher's copy (entries with teacher=True), in kernel layout; the
    DINO / iBOT centres; the optimiser's step with its two bias corrections."""
    entries = list(entries)
    spec: Dict[str, Tuple[int, ...]] = {}
    for prefix in ("param", "exp_avg", "exp_avg_sq"):
        spec.update({f"{prefix}/{e.name}": tuple(e.shape) for e in entries})
    spec.update({f"teacher/{e.name}": tuple(e.shape) for e in entries if e.teacher})
    spec["center/dino"] = spec["center/ibot"] = (int(center_dim),)
    spec["optimizer/hyper"] = (3,)
    return spec


# ---------------------------------------------------------------------------------------------------- safetensors I/O
def _write_safetensors(path: str, tensors: Mapping[str, torch.Tensor], metadata: Optional[Dict[str, str]] = None) -> int:
    """The safetensors layout (u64 header length, JSON header, raw little-endian data), streamed one tensor at a time:
    the tensors may be views of one flat device buffer and are copied to the host one by one.  fsyncs; returns the size."""
    header: Dict[str, object] = {}
    off = 0
    for name, t in tensors.items():
        if t.dtype not in _DTYPES:
            raise TypeError(f"{name}: dtype {t.dtype} is not part of the checkpoint format")
        n = t.numel() * t.element_size()
        header[name] = {"dtype": _DTYPES[t.dtype], "shape": list(t.shape), "data_offsets": [off, off + n]}
        off += n
    if metadata:
        header["__metadata__"] = dict(metadata)
    h = json.dumps(header, separators=(",", ":")).encode()
    h += b" " * (-len(h) % 8)                 # the data starts 8-byte aligned
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(h)))
        f.write(h)
        for t in tensors.values():
            f.write(memoryview(t.detach().contiguous().cpu().view(-1).numpy()).cast("B"))
        f.flush()
        os.fsync(f.fileno())
    return 8 + len(h) + off


def _fsync_dir(path: str) -> None:
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _pipeline_split(state: dict) -> Tuple[Dict[str, torch.Tensor], str]:
    """An input pipeline's state dict -> (its byte-valued entries as uint8 tensors, the rest as JSON)."""
    raw = {f"pipeline/{k}": torch.frombuffer(bytearray(v), dtype=torch.uint8) for k, v in state.items()
           if isinstance(v, (bytes, bytearray))}
    rest = {k: v for k, v in state.items() if not isinstance(v, (bytes, bytearray))}
    return raw, json.dumps(rest)


# ---------------------------------------------------------------------------------------------------- save
def save(path: str, tensors: Mapping[str, torch.Tensor], *, step: int, cuda_rng: torch.Tensor,
         pipeline: Optional[dict] = None, config: Optional[dict] = None, rank: int = 0, world: int = 1,
         process_group=None) -> None:
    """Write a checkpoint directory at `path`, atomically.  Every rank calls this: rank 0 writes `tensors` (fp32) and
    the manifest, every rank its own RNG file (`cuda_rng`: its CUDA generator state, `pipeline`: its input pipeline's
    state dict, see data.TrainBatchPipeline.state_dict).  `config` goes into the manifest for the record."""
    path = os.path.abspath(path)
    tmp = path + ".tmp"

    def barrier():
        if world > 1:
            import torch.distributed as dist
            dist.barrier(group=process_group)

    if rank == 0:
        if os.path.exists(tmp):          # left behind by an interrupted save
            shutil.rmtree(tmp)
        os.makedirs(tmp)
    barrier()
    rng_t = {"cuda_rng": cuda_rng.detach().to(torch.uint8).cpu()}
    meta = {"format": FORMAT, "rank": str(rank)}
    if pipeline is not None:
        raw, meta["pipeline"] = _pipeline_split(pipeline)
        rng_t.update(raw)
    _write_safetensors(os.path.join(tmp, rng_file(rank)), rng_t, meta)
    if rank == 0:
        for name, t in tensors.items():
            if t.dtype != torch.float32:
                raise TypeError(f"{name}: the trainer state is fp32, got {t.dtype}")
        _write_safetensors(os.path.join(tmp, STATE_FILE), tensors, {"format": FORMAT})
    barrier()                            # every rank's file is on disk
    if rank == 0:
        files = [STATE_FILE] + [rng_file(r) for r in range(world)]
        manifest = {"format": FORMAT, "version": VERSION, "step": int(step), "world_size": int(world),
                    "config": config or {}, "files": {f: os.path.getsize(os.path.join(tmp, f)) for f in files}}
        with open(os.path.join(tmp, MANIFEST), "w") as f:
            json.dump(manifest, f, indent=1, default=str)
            f.flush()
            os.fsync(f.fileno())
        _fsync_dir(tmp)
        old = None
        if os.path.exists(path):         # replace an older checkpoint of the same name
            old = path + ".old"
            if os.path.exists(old):
                shutil.rmtree(old)
            os.rename(path, old)
        os.rename(tmp, path)
        _fsync_dir(os.path.dirname(path))
        if old is not None:
            shutil.rmtree(old)
    barrier()                            # the checkpoint is in place on return, on every rank


# ---------------------------------------------------------------------------------------------------- load
def _offenders(kind: str, names: Sequence[str], limit: int = 4) -> List[str]:
    if not names:
        return []
    more = f" (+{len(names) - limit} more)" if len(names) > limit else ""
    return [f"{kind}: {', '.join(names[:limit])}{more}"]


class Checkpoint:
    """A validated checkpoint.  `tensor(name)` reads one tensor of `trainer.safetensors` (CPU); `cuda_rng` and
    `pipeline` are this rank's RNG states (None when the load skips them or the save had no pipeline)."""

    def __init__(self, path: str, manifest: dict, state, names: List[str], cuda_rng: Optional[torch.Tensor],
                 pipeline: Optional[dict]):
        self.path, self.manifest, self._state, self.names = path, manifest, state, names
        self.step = int(manifest["step"])
        self.world_size = int(manifest["world_size"])
        self.cuda_rng, self.pipeline = cuda_rng, pipeline

    def tensor(self, name: str) -> torch.Tensor:
        return self._state.get_tensor(name)


def read_manifest(path: str) -> dict:
    fn = os.path.join(path, MANIFEST)
    if not os.path.isfile(fn):
        raise ValueError(f"{path}: no {MANIFEST}, not a checkpoint (a save that did not finish leaves only {path}.tmp)")
    with open(fn) as f:
        try:
            m = json.load(f)
        except json.JSONDecodeError as e:
            raise ValueError(f"{fn}: unreadable manifest ({e})") from None
    if m.get("format") != FORMAT or m.get("version") != VERSION:
        raise ValueError(f"{fn}: format {m.get('format')!r} version {m.get('version')!r}, expected {FORMAT!r} {VERSION}")
    return m


def load(path: str, spec: Mapping[str, Tuple[int, ...]], *, rank: int = 0, world: int = 1, rng: bool = True,
         pipeline: bool = False) -> Checkpoint:
    """Open and validate the checkpoint at `path` against `spec` (state_spec of the loading trainer).  Raises ValueError
    naming the first offending entries when the manifest is missing, a file has another size than the manifest states,
    a tensor of `spec` is missing or has another shape or dtype, or the file holds a name `spec` does not.  With `rng`,
    this rank's RNG file is read too, and the checkpoint must come from a job of `world` ranks; with `pipeline`, it must
    hold an input pipeline's state."""
    from safetensors import safe_open

    if pipeline and not rng:
        raise ValueError("an input pipeline's state is part of the per-rank RNG state: it needs rng=True")
    path = os.path.abspath(path)
    m = read_manifest(path)
    bad = []
    for f, size in m["files"].items():
        fn = os.path.join(path, f)
        got = os.path.getsize(fn) if os.path.isfile(fn) else None
        if got != size:
            bad.append(f"{f} ({'missing' if got is None else f'{got} B'}, manifest {size} B)")
    if bad:
        raise ValueError(f"{path}: files do not match the manifest: " + "; ".join(bad[:4]))
    if rng and int(m["world_size"]) != world:
        raise ValueError(f"{path}: saved by {m['world_size']} rank(s), loading on {world}: the per-rank RNG streams do not "
                         f"carry over; load with rng=False to resume on another number of GPUs")
    st = safe_open(os.path.join(path, STATE_FILE), framework="pt", device="cpu")
    names = list(st.keys())
    have = set(names)
    missing = [n for n in spec if n not in have]
    unexpected = [n for n in names if n not in spec]
    wrong = []
    for n in spec:
        if n in have:
            sl = st.get_slice(n)
            shape, dtype = tuple(sl.get_shape()), sl.get_dtype()
            if shape != tuple(spec[n]) or dtype != "F32":
                wrong.append(f"{n} {dtype}{list(shape)} (expected F32{list(spec[n])})")
    problems = _offenders("wrong shape", wrong) + _offenders("missing", missing) + _offenders("unexpected", unexpected)
    if problems:
        raise ValueError(f"{path}: checkpoint does not match this trainer: " + "; ".join(problems))
    cuda_rng = pipe = None
    if rng:
        fn = os.path.join(path, rng_file(rank))
        with safe_open(fn, framework="pt", device="cpu") as r:
            keys = set(r.keys())
            if "cuda_rng" not in keys:
                raise ValueError(f"{fn}: no cuda_rng tensor")
            cuda_rng = r.get_tensor("cuda_rng")
            meta = r.metadata() or {}
            if "pipeline" in meta:
                pipe = json.loads(meta["pipeline"])
                pipe.update({k[len("pipeline/"):]: bytes(r.get_tensor(k).numpy()) for k in keys if k.startswith("pipeline/")})
        if pipeline and pipe is None:
            raise ValueError(f"{fn}: the checkpoint was saved without an input pipeline state")
    return Checkpoint(path, m, st, names, cuda_rng, pipe)
