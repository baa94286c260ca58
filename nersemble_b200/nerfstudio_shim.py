"""Minimal duck-typed stand-ins for the nerfstudio types on the plugin surface.

Used ONLY when the real `nerfstudio` package is not importable (it is not installed in this
image); with nerfstudio present the plugin classes use its own RayBundle / RaySamples / Frustums /
FieldHeadNames / Model / TrainingCallback so they drop in under scripts/train/train_nersemble.py.
Semantics follow nerfstudio 0.3.1 (cameras/rays.py, engine/callbacks.py, models/base_model.py).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from enum import Enum, auto
from typing import Any, Dict, List, Optional, Type

import torch
from torch import nn

try:  # pragma: no cover - real nerfstudio is not installed in this image
    from nerfstudio.cameras.rays import Frustums, RayBundle, RaySamples  # type: ignore
    from nerfstudio.engine.callbacks import (TrainingCallback, TrainingCallbackAttributes,  # type: ignore
                                             TrainingCallbackLocation)
    from nerfstudio.field_components.field_heads import FieldHeadNames  # type: ignore
    from nerfstudio.models.base_model import Model  # type: ignore
    HAVE_NERFSTUDIO = True
except Exception:  # noqa: BLE001
    HAVE_NERFSTUDIO = False

    class _Bag:
        def __len__(self):
            return self.shape[0]

    class Frustums(_Bag):
        def __init__(self, origins, directions, starts, ends, pixel_area, offsets=None):
            self.origins, self.directions, self.starts, self.ends = origins, directions, starts, ends
            self.pixel_area, self.offsets = pixel_area, offsets

        @property
        def shape(self):
            return self.origins.shape[:-1]

        def get_positions(self):
            pos = self.origins + self.directions * (self.starts + self.ends) / 2
            return pos if self.offsets is None else pos + self.offsets

        def set_offsets(self, offsets):
            self.offsets = offsets

    class RaySamples(_Bag):
        def __init__(self, frustums, camera_indices=None, deltas=None, metadata=None, times=None):
            self.frustums, self.camera_indices, self.deltas = frustums, camera_indices, deltas
            self.metadata, self.times = metadata, times

        @property
        def shape(self):
            return self.frustums.shape

    class RayBundle(_Bag):
        def __init__(self, origins, directions, pixel_area=None, camera_indices=None, nears=None, fars=None,
                     metadata=None, times=None):
            self.origins, self.directions, self.pixel_area = origins, directions, pixel_area
            self.camera_indices, self.nears, self.fars = camera_indices, nears, fars
            self.metadata = metadata if metadata is not None else {}
            self.times = times

        @property
        def shape(self):
            return self.origins.shape[:-1]

        def get_row_major_sliced_ray_bundle(self, start, end):
            def sl(t):
                return None if t is None else t.reshape(-1, t.shape[-1])[start:end]
            return RayBundle(sl(self.origins), sl(self.directions), sl(self.pixel_area), sl(self.camera_indices),
                             sl(self.nears), sl(self.fars), {k: sl(v) for k, v in self.metadata.items()}, sl(self.times))

    class FieldHeadNames(Enum):
        RGB = "rgb"
        DENSITY = "density"
        NORMALS = "normals"

    class TrainingCallbackLocation(Enum):
        BEFORE_TRAIN_ITERATION = auto()
        AFTER_TRAIN_ITERATION = auto()

    @dataclass
    class TrainingCallbackAttributes:
        optimizers: Any = None
        grad_scaler: Any = None
        pipeline: Any = None

    class TrainingCallback:
        def __init__(self, where_to_run, func, update_every_num_iters=None, iters=None, args=None, kwargs=None):
            self.where_to_run, self.func = where_to_run, func
            self.update_every_num_iters, self.iters = update_every_num_iters, iters
            self.args = args if args is not None else []
            self.kwargs = kwargs if kwargs is not None else {}

        def run_callback(self, step: int):
            if self.update_every_num_iters is not None:
                if step % self.update_every_num_iters == 0:
                    self.func(*self.args, **self.kwargs, step=step)
            elif self.iters is not None and step in self.iters:
                self.func(*self.args, **self.kwargs, step=step)

        def run_callback_at_location(self, step, location):
            if location in self.where_to_run:
                self.run_callback(step)


    class Model(nn.Module):
        """nerfstudio.models.base_model.Model (0.3.1): constructor protocol, device, forward, the chunked camera-ray
        render, checkpoint loading and the step hook -- what the trainer / pipeline call on a model."""

        def __init__(self, config, scene_box, num_train_data: int, **kwargs):
            super().__init__()
            self.config = config
            self.scene_box = scene_box
            self.render_aabb = None
            self.num_train_data = num_train_data
            self.kwargs = kwargs
            self.collider = None
            self.populate_modules()
            self.callbacks = None
            self.device_indicator_param = nn.Parameter(torch.empty(0))

        @property
        def device(self):
            return self.device_indicator_param.device

        def populate_modules(self):
            pass

        def get_training_callbacks(self, training_callback_attributes):
            return []

        def forward(self, ray_bundle):
            if self.collider is not None:
                ray_bundle = self.collider(ray_bundle)
            return self.get_outputs(ray_bundle)

        @torch.no_grad()
        def get_outputs_for_camera_ray_bundle(self, camera_ray_bundle):
            n = self.config.eval_num_rays_per_chunk
            h, w = camera_ray_bundle.origins.shape[:2]
            lists: Dict[str, list] = {}
            for i in range(0, h * w, n):
                rb = camera_ray_bundle.get_row_major_sliced_ray_bundle(i, i + n)
                for name, out in self.forward(ray_bundle=rb).items():
                    if torch.is_tensor(out):          # tuple-wrapped per-sample outputs are skipped (NeRSemble wraps them)
                        lists.setdefault(name, []).append(out)
            return {k: torch.cat(v).view(h, w, -1) for k, v in lists.items()}

        def load_model(self, loaded_state: Dict[str, Any]) -> None:
            state = {key.replace("module.", ""): value for key, value in loaded_state["model"].items()}
            self.load_state_dict(state)

        def update_to_step(self, step: int) -> None:
            """Called when loading a checkpoint to fast-forward step-dependent state (schedulers)."""


class SceneBox:
    def __init__(self, aabb: torch.Tensor):
        self.aabb = aabb
