"""Data pipeline: fake ImageNet, ImageFolder + transforms, distributed sampling and a pinned,
double-buffered host->device prefetcher.

Reference: ``build_datasets`` (run_vit_training.py:30-96), ``FakeImageNetDataset`` (utils.py:46-55) and
``pl.MpDeviceLoader`` (background host->device transfer, :74,88).
"""
from __future__ import annotations

import os
from typing import Iterator, Tuple

import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.distributed import DistributedSampler

IMAGENET_TRAIN_LEN = 1281167  # run_vit_training.py:59
IMAGENET_VAL_LEN = 50000      # run_vit_training.py:60


class FakeImageNetDataset(Dataset):
    """All-zero images with label 0 (the loss must collapse to ~0: a built-in sanity signal)."""

    def __init__(self, image_size: int, length: int):
        self.image_size = image_size
        self.length = length

    def __getitem__(self, idx):
        return torch.zeros(3, self.image_size, self.image_size), 0

    def __len__(self) -> int:
        return self.length

    def __repr__(self) -> str:
        return f"FakeImageNetDataset(image_size={self.image_size}, length={self.length})"


class FakeBatchLoader:
    """Fast path for ``--fake_data``: the batch is constant, so skip worker processes and collation and
    serve one pinned host batch repeatedly (still copied host->device every step by the prefetcher)."""

    def __init__(self, image_size: int, local_batch: int, num_batches: int, pin: bool):
        self.images = torch.zeros(local_batch, 3, image_size, image_size)
        self.target = torch.zeros(local_batch, dtype=torch.long)
        if pin:
            self.images = self.images.pin_memory()
            self.target = self.target.pin_memory()
        self.num_batches = num_batches

    def __iter__(self):
        for _ in range(self.num_batches):
            yield self.images, self.target

    def __len__(self) -> int:
        return self.num_batches


class DevicePrefetcher:
    """Iterates a host loader and keeps ``depth`` batches in flight on a dedicated copy stream
    (pinned memory + non_blocking copies), the CUDA analogue of ``pl.MpDeviceLoader``."""

    def __init__(self, loader, device: torch.device, depth: int = 2):
        self.loader, self.device, self.depth = loader, device, max(1, depth)
        self.cuda = device.type == "cuda"
        self.stream = torch.cuda.Stream(device=device) if self.cuda else None

    def __len__(self) -> int:
        return len(self.loader)

    def _stage(self, batch):
        images, target = batch
        if not self.cuda:
            return images, torch.as_tensor(target), None
        with torch.cuda.stream(self.stream):
            if not images.is_pinned():
                images = images.pin_memory()
            target = torch.as_tensor(target)
            if not target.is_pinned():
                target = target.pin_memory()
            d_img = images.to(self.device, non_blocking=True)
            d_tgt = target.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return d_img, d_tgt, ev

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        it = iter(self.loader)
        queue = []
        for _ in range(self.depth):
            try:
                queue.append(self._stage(next(it)))
            except StopIteration:
                break
        while queue:
            d_img, d_tgt, ev = queue.pop(0)
            try:
                queue.append(self._stage(next(it)))
            except StopIteration:
                pass
            if ev is not None:
                torch.cuda.current_stream().wait_event(ev)
                d_img.record_stream(torch.cuda.current_stream())
                d_tgt.record_stream(torch.cuda.current_stream())
            yield d_img, d_tgt


def _image_folder_datasets(cfg):
    import torchvision
    import torchvision.transforms as T

    train_transform = T.Compose([
        T.RandomResizedCrop(cfg.image_size, interpolation=T.InterpolationMode.BICUBIC),
        T.RandomHorizontalFlip(),
        T.ToTensor(),
        T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]),
    ])
    val_transform = T.Compose([
        T.Resize((cfg.image_size * 256) // 224, interpolation=T.InterpolationMode.BICUBIC),
        T.CenterCrop(cfg.image_size),
        T.ToTensor(),
        T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]),
    ])
    train = torchvision.datasets.ImageFolder(os.path.join(cfg.data_dir, "train"), train_transform)
    val = torchvision.datasets.ImageFolder(os.path.join(cfg.data_dir, "val"), val_transform)
    return train, val


def build_datasets(cfg, device: torch.device, world_size: int, rank: int, log=print):
    """Returns (train_dataset, train_loader, train_sampler, val_dataset, val_loader, val_sampler)."""
    assert cfg.batch_size % world_size == 0, "global batch size must be divisible by the world size"  # :34
    local_batch_size = cfg.batch_size // world_size
    pin = device.type == "cuda"
    if not cfg.fake_data:
        log(f"loading images from directory: {cfg.data_dir}")
        train_dataset, val_dataset = _image_folder_datasets(cfg)
    else:
        log("loading fake images")
        train_dataset = FakeImageNetDataset(cfg.image_size, IMAGENET_TRAIN_LEN)
        val_dataset = FakeImageNetDataset(cfg.image_size, IMAGENET_VAL_LEN)

    train_sampler = DistributedSampler(train_dataset, num_replicas=world_size, rank=rank, drop_last=True, shuffle=True)
    val_sampler = DistributedSampler(val_dataset, num_replicas=world_size, rank=rank, drop_last=True, shuffle=False)
    if cfg.fake_data:
        # identical contents to DataLoader(FakeImageNetDataset) with drop_last=True, without the worker overhead
        train_loader = FakeBatchLoader(cfg.image_size, local_batch_size, len(train_sampler) // local_batch_size, pin)
        val_loader = FakeBatchLoader(cfg.image_size, local_batch_size, len(val_sampler) // local_batch_size, pin)
    else:
        workers = cfg.num_workers
        kw = dict(batch_size=local_batch_size, drop_last=True, num_workers=workers, pin_memory=pin,
                  persistent_workers=workers > 0)  # the reference crashes with --num_workers 0 (:72); guarded here
        train_loader = DataLoader(train_dataset, sampler=train_sampler, **kw)
        val_loader = DataLoader(val_dataset, sampler=val_sampler, **kw)
    depth = getattr(cfg, "h2d_prefetch", 2)
    train_loader = DevicePrefetcher(train_loader, device, depth)
    val_loader = DevicePrefetcher(val_loader, device, depth)
    return train_dataset, train_loader, train_sampler, val_dataset, val_loader, val_sampler
