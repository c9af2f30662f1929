"""Sampler state and orchestration with the V x T latent grid resident on the device (SURVEY.md section 8f row 2).

Host-side mirror of the reference's ``SlidingIterativeSampler`` (SAMP = src/samplers/sliding_iterative_sampler.py):
same constructor arguments, label formatting, argument checks (SAMP:72-90, same messages), task lists (SAMP:192-199),
sample loading (SAMP:102-153) and bookkeeping (SAMP:181-185).  What changes is where the state lives:

* the reference keeps ``latents[spa][tem]`` / ``timestep_indices[spa][tem]`` as nested Python dicts of CPU tensors behind a
  ``threading.Lock`` and moves every latent device -> host -> device around every task (``latent.cpu()`` +
  ``timestep_index.item()`` per grid cell, SAMP:181-185);
* here the grid is two device tensors (``[V, T, 4, h, w]`` and ``[V, T]`` int64); a task gathers its rows with one advanced
  index and scatters its result with one ``index_put`` -- no host synchronisation, no per-cell Python.

Multi-GPU (one process per GPU, SURVEY 8e row 1): the tasks of a round are independent, so rank r runs
``sharding.shard_tasks(len(tasks), r, world)`` and the ranks exchange the updated cells with one all-gather per round
(``sharding.exchange_grid_updates``) instead of the reference's shared dict + lock + thread-per-GPU queue
(src/samplers/sampling_runner.py:26-43).  Pinned against the reference sampler run end to end on stubs
(tests/golden/gen_golden.py::gen_sampler -> tests/test_sampler.py).  Alternatively (``execute_tasks(frame_sharded=True)``
with a ``sharded.FrameShardedPipeline``) every rank runs every task with each window split over the ranks by frames, which
keeps all GPUs busy when a round has fewer tasks than GPUs (DESIGN.md section 7); ``execute_tasks(cfg_split=True)`` with a
``cfg_split.CFGSplitPipeline`` does the same with each window step split by CFG half over two ranks (or, with a
``cfg_split.CFGGridPipeline``, by CFG half and frames over 2R ranks).

The dataset object supplies ``scene_label`` and ``get_item(scene_label, spa_labels, tem_labels, input_spa_labels)`` exactly
like the reference's ``SpaTemDataset`` (src/data/spatem_dataset.py:76-212); pipelines supply
``sliding_iterative_denoise(**kwargs) -> {"images", "latents", "timestep_indices", "fully_denoised"}`` (PIPE:439-559), e.g.
``B200Diffuman4DPipeline``.

Input prefetch and asynchronous output (SURVEY 8f rows 3 and 4, both opt-in): in the reference every worker thread runs
``dataset.get_item`` (PIL decode, crop, bicubic resize, composite, Pluecker rays: CPU work) -> denoise ->
``save_sampling_results`` (webp grid + per-image JPEG, src/samplers/utils/sampling_utils.py:54-114) strictly in sequence, so
the GPU idles during both.  With ``prefetch=True`` the dataset part of the NEXT task of the round is loaded by a helper
thread while the current task is on the GPU (the tasks of a round touch disjoint target cells, and the grid rows of a task
are still gathered on the calling thread right before its denoise); with ``async_save=True`` ``save_fn`` runs on one
worker thread in task order behind a bounded queue and its first exception is re-raised by ``execute_tasks``.

Encoded-image cache (SURVEY 8f row 1, first step; opt-in ``cache_pixel_latents=True``): the reference VAE-encodes all frames
of a task in every task (PIPE:208-214), i.e. every image of the grid once per round and the cond view of a temporal task T
times more.  With the cache the encoded image latents live in a third device grid ``[V, T, 4, h, w]``; a task encodes only
the cells not seen before and hands ``pixel_values_latents`` to the pipeline.  Note the semantics: the reference draws
``latent_dist.sample()`` anew at every encode, the cache keeps the first draw of a cell for the whole run.
"""
from __future__ import annotations

import queue
import threading
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from .sharding import exchange_grid_updates, shard_tasks


class B200SlidingIterativeSampler:
    def __init__(self, dataset, pipelines: Sequence, output_dir: Optional[str] = "./results/debug",
                 window_size: int = 12, sliding_stride: int = 1, sliding_shift: int = 0, bidirectional: bool = True,
                 num_denoising_steps: int = 1, alternation_rounds: int = 3, guidance_scale: float = 2.0,
                 spa_label_range: Optional[List[int]] = (0, 48, 1), tem_label_range: Optional[List[int]] = (0, 150, 1),
                 spa_labels: Optional[Sequence[int]] = None, tem_labels: Optional[Sequence[int]] = None,
                 input_spa_labels: Sequence[int] = (1, 13, 25, 37),
                 save_fn: Optional[Callable[[dict, Optional[str]], None]] = None, prefetch: bool = False,
                 async_save: bool = False, cache_pixel_latents: bool = False):
        self.dataset, self.pipelines, self.output_dir, self.save_fn = dataset, list(pipelines), output_dir, save_fn
        self.prefetch, self.async_save, self.cache_pixel_latents = prefetch, async_save, cache_pixel_latents
        self.grid_pixel_latents: Optional[torch.Tensor] = None      # [V, T, C, h, w] encoded images (cache_pixel_latents)
        self._pixel_cached: set = set()                             # (view, frame) cells already encoded (host-side: no sync)
        self.vae_images_encoded = 0                                 # images sent through the VAE encoder by the cache path
        self.window_size, self.sliding_stride, self.sliding_shift = window_size, sliding_stride, sliding_shift
        self.bidirectional, self.num_denoising_steps = bidirectional, num_denoising_steps
        self.alternation_rounds, self.guidance_scale = alternation_rounds, guidance_scale

        if spa_labels is not None:                                                    # SAMP:49-64
            self.spa_labels = [f"{int(i):02d}" for i in spa_labels]
        elif spa_label_range is not None:
            b, e, s = spa_label_range
            self.spa_labels = [f"{int(i):02d}" for i in range(b, e, s)]
        else:
            raise ValueError("spa_labels or spa_label_range must be provided")
        if tem_labels is not None:
            self.tem_labels = [f"{int(i):06d}" for i in tem_labels]
        elif tem_label_range is not None:
            b, e, s = tem_label_range
            self.tem_labels = [f"{int(i):06d}" for i in range(b, e, s)]
        else:
            raise ValueError("tem_labels or tem_label_range must be provided")
        self.input_spa_labels = [f"{int(i):02d}" for i in input_spa_labels]
        self.target_spa_labels = [label for label in self.spa_labels if label not in self.input_spa_labels]

        if self.window_size > len(self.target_spa_labels):                            # SAMP:72-90
            raise ValueError(
                f"window_size(={self.window_size}) must be <= len(target_spa_labels)(={len(self.target_spa_labels)})")
        if len(self.target_spa_labels) % self.sliding_stride != 0:
            raise ValueError(
                f"len(target_spa_labels)(={len(self.target_spa_labels)}) % sliding_stride(={self.sliding_stride}) must be 0")
        if len(self.tem_labels) % self.sliding_stride != 0:
            raise ValueError(f"len(tem_labels)(={len(self.tem_labels)}) % sliding_stride(={self.sliding_stride}) must be 0")
        if self.alternation_rounds > 1 and self.window_size > len(self.tem_labels):
            raise ValueError(f"window_size(={self.window_size}) must be <= the number of tem_labels(={len(self.tem_labels)}) "
                             "when alternation_rounds > 1")

        # spatio-temporal grid (SAMP:92-98): device tensors, allocated when the first task result arrives
        self._spa_index = {label: i for i, label in enumerate(self.spa_labels)}
        self._tem_index = {label: i for i, label in enumerate(self.tem_labels)}
        self.grid_latents: Optional[torch.Tensor] = None            # [V, T, C, h, w]
        self.grid_timestep_indices: Optional[torch.Tensor] = None   # [V, T] int64
        self._grid_device: Optional[torch.device] = None
        self.prepare_tasks()

    # ---- grid -------------------------------------------------------------------------------------------------
    def _cells(self, labels) -> Tuple[torch.Tensor, torch.Tensor]:
        vi = torch.tensor([self._spa_index[s] for _, s, _ in labels], dtype=torch.int64)
        ti = torch.tensor([self._tem_index[t] for _, _, t in labels], dtype=torch.int64)
        return vi, ti

    def _ensure_grid(self, like: torch.Tensor):
        if self.grid_latents is None:
            V, T = len(self.spa_labels), len(self.tem_labels)
            self._grid_device = like.device
            self.grid_latents = torch.zeros((V, T, *like.shape[1:]), dtype=like.dtype, device=like.device)
            self.grid_timestep_indices = torch.zeros((V, T), dtype=torch.int64, device=like.device)

    def latent(self, spa_label: str, tem_label: str) -> Optional[torch.Tensor]:
        """Grid cell accessor with the reference's ``sampler.latents[spa][tem]`` meaning (None until written)."""
        if self.grid_latents is None:
            return None
        return self.grid_latents[self._spa_index[spa_label], self._tem_index[tem_label]]

    def timestep_index(self, spa_label: str, tem_label: str) -> int:
        if self.grid_timestep_indices is None:
            return 0
        return int(self.grid_timestep_indices[self._spa_index[spa_label], self._tem_index[tem_label]])

    # ---- SAMP:102-153 -----------------------------------------------------------------------------------------
    def load_sample(self, alt: int, domain: str, domain_label: str) -> dict:
        return self._attach_grid(self._fetch(alt, domain, domain_label))

    def _fetch(self, alt: int, domain: str, domain_label: str) -> dict:
        """The dataset half of SAMP:102-153 (host work only: safe on a helper thread)."""
        if domain == "spatial":
            spa_labels, tem_labels = self.spa_labels, [domain_label]
            input_indices = torch.tensor([self.spa_labels.index(label) for label in self.input_spa_labels])
            target_indices = torch.tensor([self.spa_labels.index(label) for label in self.target_spa_labels])
        elif domain == "temporal":
            spa_labels, tem_labels = [domain_label], self.tem_labels
            half = len(self.tem_labels)   # first half is input, second half is target
            input_indices = torch.tensor(list(range(half)))
            target_indices = torch.tensor(list(range(half, 2 * half)))
        else:
            raise ValueError(f"Invalid domain: {domain}")
        sample = self.dataset.get_item(scene_label=self.dataset.scene_label, spa_labels=spa_labels, tem_labels=tem_labels,
                                       input_spa_labels=self.input_spa_labels)
        sample.update(alt=alt, domain=domain, domain_label=domain_label, input_indices=input_indices,
                      target_indices=target_indices)
        cond_masks = sample["cond_masks"]
        cond_masks[...] = 1.0
        cond_masks[input_indices, ...] = 0.0
        sample["cond_masks"] = cond_masks
        return sample

    def _attach_grid(self, sample: dict) -> dict:
        """The grid half: this task's rows of the latent / timestep grid (reads what earlier ROUNDS wrote)."""
        target_indices = sample["target_indices"]
        vi, ti = self._cells(sample["labels"])
        sample["_cells"] = (vi, ti)
        if self.grid_latents is None:
            sample["timestep_indices"] = torch.zeros(len(sample["labels"]), dtype=torch.int64)
            sample["latents"] = None
        else:
            dev = self._grid_device
            tidx = self.grid_timestep_indices[vi.to(dev), ti.to(dev)]
            sample["timestep_indices"] = tidx
            # one host read per TASK (the reference reads every cell): fresh targets start from noise inside the pipeline
            fresh = int(tidx[target_indices[0]]) == 0
            sample["latents"] = None if fresh else self.grid_latents[vi.to(dev), ti.to(dev)]
        return sample

    # ---- SAMP:155-190 -----------------------------------------------------------------------------------------
    @torch.no_grad()
    def denoise(self, sample: dict, pipe_idx: int = 0) -> dict:
        pipeline = self.pipelines[pipe_idx]
        extra = {}
        if self.cache_pixel_latents and getattr(pipeline, "vae", None) is not None:
            extra["pixel_values_latents"] = self._cached_pixel_latents(sample, pipeline)
        result = pipeline.sliding_iterative_denoise(
            pixel_values=None if extra else sample["pixel_values"], plucker_embeds=sample["plucker_embeds"],
            skeletons=sample["skeletons"],
            cond_masks=sample["cond_masks"], latents=sample["latents"], domain=sample["domain"],
            timestep_indices=sample["timestep_indices"], window_size=self.window_size, sliding_stride=self.sliding_stride,
            sliding_shift=self.sliding_shift, bidirectional=self.bidirectional,
            num_denoising_steps=self.num_denoising_steps, alternation_rounds=self.alternation_rounds,
            guidance_scale=self.guidance_scale, **extra)
        lat = result["latents"]
        self._ensure_grid(lat)
        vi, ti = (t.to(self._grid_device) for t in sample["_cells"])
        self.grid_latents.index_put_((vi, ti), lat.to(self.grid_latents.dtype))
        self.grid_timestep_indices.index_put_((vi, ti), result["timestep_indices"].to(torch.int64))
        sample["images"] = result.get("images")
        sample["timestep_indices"] = result["timestep_indices"]
        sample["fully_denoised"] = result["fully_denoised"]
        sample["result_latents"] = lat
        return sample

    def _cached_pixel_latents(self, sample: dict, pipeline) -> torch.Tensor:
        """Encoded images of this task's cells: encode what the cache has not seen (PIPE:208-214 encodes everything)."""
        vi, ti = sample["_cells"]
        keys = list(zip(vi.tolist(), ti.tolist()))
        missing = [k for k, key in enumerate(keys) if key not in self._pixel_cached]
        dev = pipeline.device
        if missing:
            px = sample["pixel_values"][torch.tensor(missing)].to(dev, torch.bfloat16)
            enc = pipeline.vae.encode_latents(px)
            self.vae_images_encoded += len(missing)
            if self.grid_pixel_latents is None:
                V, T = len(self.spa_labels), len(self.tem_labels)
                self.grid_pixel_latents = torch.zeros((V, T, *enc.shape[1:]), dtype=enc.dtype, device=enc.device)
            mv, mt = vi[missing].to(enc.device), ti[missing].to(enc.device)
            self.grid_pixel_latents.index_put_((mv, mt), enc)
            self._pixel_cached.update(keys[k] for k in missing)
        g = self.grid_pixel_latents
        return g[vi.to(g.device), ti.to(g.device)]

    # ---- SAMP:192-214 -----------------------------------------------------------------------------------------
    def prepare_tasks(self):
        domains = (["spatial", "temporal"] * self.alternation_rounds)[: self.alternation_rounds]
        self.all_tasks: List[List[Dict]] = []
        for i, domain in enumerate(domains):
            domain_labels = self.tem_labels if domain == "spatial" else self.target_spa_labels
            self.all_tasks.append([{"alt": i + 1, "domain": domain, "domain_label": label} for label in domain_labels])

    def execute_one_task(self, task: dict, pipe_idx: int = 0) -> dict:
        sample = self.denoise(self.load_sample(**task), pipe_idx=pipe_idx)
        if self.save_fn is not None:
            self.save_fn(sample, self.output_dir)
        return sample

    def execute_tasks(self, rank: int = 0, world: int = 1, group=None, pipe_idx: int = 0, frame_sharded: bool = False,
                      cfg_split: bool = False):
        """All rounds.  ``world > 1`` (inside an initialised ``torch.distributed`` job): this rank runs its share of every
        round, then the ranks all-gather the cells they updated (the round barrier of RUN:53-55).

        ``frame_sharded=True``: ``pipelines[pipe_idx]`` is a ``FrameShardedPipeline`` and every rank of its process group
        runs every task, each window split over the ranks by frames.  Every rank's grid ends up identical, so there is no
        per-round exchange; ``rank`` / ``world`` / ``group`` are not used (the pipeline's group defines the ranks), and
        ``save_fn`` runs on the pipeline's rank 0 only.

        ``cfg_split=True``: the same, with a ``cfg_split.CFGSplitPipeline`` whose ranks each run one CFG half of every
        window step, or a ``cfg_split.CFGGridPipeline`` whose ranks each run a frame shard of one CFG half."""
        save_fn = self.save_fn
        if frame_sharded and cfg_split:
            raise ValueError("frame_sharded and cfg_split are two different multi-GPU modes; pass one of them")
        if frame_sharded or cfg_split:
            from .cfg_split import CFGSplitPipeline
            from .sharded import FrameShardedPipeline
            pipe = self.pipelines[pipe_idx]
            cls = FrameShardedPipeline if frame_sharded else CFGSplitPipeline
            if not isinstance(pipe, cls):
                raise ValueError(f"{'frame_sharded' if frame_sharded else 'cfg_split'}=True needs a {cls.__name__} in "
                                 "pipelines[pipe_idx]")
            rank, world, save_fn = 0, 1, (save_fn if pipe.rank == 0 else None)
        saver = _AsyncSaver(save_fn, self.output_dir) if (self.async_save and save_fn is not None) else None
        try:
            for tasks in self.all_tasks:
                mine = list(shard_tasks(len(tasks), rank, world) if world > 1 else range(len(tasks)))
                keys, lats, tis = [], [], []
                fetched = _Prefetcher(self._fetch, [tasks[i] for i in mine]) if self.prefetch else None
                for n, i in enumerate(mine):
                    raw = fetched.get(n) if fetched is not None else self._fetch(**tasks[i])
                    sample = self.denoise(self._attach_grid(raw), pipe_idx=pipe_idx)
                    if saver is not None:
                        saver.submit(sample)
                    elif save_fn is not None:
                        save_fn(sample, self.output_dir)
                    if world > 1:
                        vi, ti = sample["_cells"]
                        keys += list(zip(vi.tolist(), ti.tolist()))
                        lats.append(sample["result_latents"])
                        tis.append(sample["timestep_indices"].to(torch.int64))
                if world > 1:
                    self._exchange(keys, lats, tis, group)
        finally:
            if saver is not None:
                saver.close()

    def _exchange(self, keys, lats, tis, group):
        if lats:
            lat, ti = torch.cat(lats), torch.cat(tis)
        else:   # a rank without tasks in this round still takes part in the collective
            ref = self.grid_latents
            if ref is None:
                raise RuntimeError("a rank with no task in the first round cannot size the exchange buffers; "
                                   "use world <= number of tasks per round")
            lat, ti = ref.new_zeros((0, *ref.shape[2:])), torch.zeros(0, dtype=torch.int64, device=ref.device)
        self._ensure_grid(lat)
        merged = exchange_grid_updates(keys, lat, ti, group=group)
        if merged:
            cells = list(merged.keys())
            vi = torch.tensor([c[0] for c in cells], dtype=torch.int64, device=self._grid_device)
            tj = torch.tensor([c[1] for c in cells], dtype=torch.int64, device=self._grid_device)
            self.grid_latents.index_put_((vi, tj), torch.stack([merged[c][0] for c in cells]).to(self.grid_latents.dtype))
            self.grid_timestep_indices.index_put_(
                (vi, tj), torch.tensor([merged[c][1] for c in cells], dtype=torch.int64, device=self._grid_device))


class _Prefetcher:
    """Loads item n + 1 of a task list on a helper thread while the caller works on item n (depth 1: one sample of a
    48-view task is ~0.6 GB of host tensors at 1024^2)."""

    def __init__(self, fetch: Callable[..., dict], tasks: List[dict]):
        self._fetch, self._tasks = fetch, tasks
        self._next: Optional[Tuple[int, threading.Thread, list]] = None
        self._start(0)

    def _start(self, n: int):
        if n >= len(self._tasks):
            self._next = None
            return
        box: list = []

        def run():
            try:
                box.append((True, self._fetch(**self._tasks[n])))
            except BaseException as e:  # noqa: BLE001 -- handed to the consumer
                box.append((False, e))
        t = threading.Thread(target=run, name="d4d-prefetch", daemon=True)
        t.start()
        self._next = (n, t, box)

    def get(self, n: int) -> dict:
        assert self._next is not None and self._next[0] == n, "tasks are consumed in order"
        _, t, box = self._next
        t.join()
        self._start(n + 1)
        ok, val = box[0]
        if not ok:
            raise val
        return val


class _AsyncSaver:
    """``save_fn(sample, output_dir)`` on one worker thread, in submission order, at most ``depth`` samples waiting.  The
    first exception stops further saves and is re-raised by ``submit`` / ``close``."""

    def __init__(self, save_fn: Callable[[dict, Optional[str]], None], output_dir: Optional[str], depth: int = 2):
        self._save_fn, self._output_dir = save_fn, output_dir
        self._q: "queue.Queue" = queue.Queue(maxsize=depth)
        self._error: Optional[BaseException] = None
        self._thread = threading.Thread(target=self._run, name="d4d-save", daemon=True)
        self._thread.start()

    def _run(self):
        while True:
            sample = self._q.get()
            if sample is None:
                return
            if self._error is None:
                try:
                    self._save_fn(sample, self._output_dir)
                except BaseException as e:  # noqa: BLE001 -- re-raised on the caller's thread
                    self._error = e

    def submit(self, sample: dict):
        if self._error is not None:
            raise self._error
        self._q.put(sample)

    def close(self):
        self._q.put(None)
        self._thread.join()
        if self._error is not None:
            raise self._error
