"""hyperreel_b200 -- H100-native drop-in for HyperReel's per-ray rendering hot path.

Operator surface (same names as the reference's ``nlf`` package, SURVEY.md section 8b):
``render_fn_dict`` / ``RenderLightfield`` / ``render_chunked`` (rendering.py), ``model_dict`` /
``LightfieldModel`` (models.py), ``INRSystem`` (system.py); training batches generated on the device from the
training images: ``DeviceRayBatches`` (train_data.py); decoded frames
resized to the training resolution as the datasets' ``get_rgb`` resizes them: ``resize_frames`` / ``dataset_frames`` (resize.py); a scene directory's views as the datasets' loaders build them: ``dataset_cameras`` (datasets.py); one training run of a config from a scene directory, in the reference's order and with resumable checkpoints: ``fit`` (fit.py).  All compute is in ``libhyperreel_b200.so`` (csrc/, sm_90a CUDA behind the C-ABI of include/hyperreel_b200.h).
"""
from . import camera, configs, datasets, lightfield, metrics, rays, resize, train_data  # noqa: F401
from .camera import (Camera, TwoPlaneCamera, VisualRequest, embedding_requests, generate_rays, render_embeddings,  # noqa: F401
                     render_video, score_views, spiral_path)
from .lightfield import lightfield_cameras, stanford_file_coords  # noqa: F401
from .datasets import DatasetViews, FrameSource, dataset_cameras  # noqa: F401
from .config import Cfg, epochs_to_iters, load_model_yaml, to_cfg  # noqa: F401
from .models import LightfieldModel, model_dict  # noqa: F401
from .resize import dataset_frames, resize_frames  # noqa: F401
from .rendering import RenderLightfield, render_chunked, render_fn_dict  # noqa: F401
from .signature import Signature, UnsupportedPipeline, lower  # noqa: F401
from .system import INRSystem  # noqa: F401
from .train_data import DeviceRayBatches, importance_subsample_plan, regular_subsample_plan  # noqa: F401
from .fit import fit  # noqa: F401

__all__ = ["camera", "Camera", "TwoPlaneCamera", "generate_rays", "render_video", "score_views", "render_embeddings", "embedding_requests", "VisualRequest", "spiral_path", "lightfield", "lightfield_cameras",
           "stanford_file_coords", "datasets", "dataset_cameras", "DatasetViews", "FrameSource", "resize", "resize_frames", "dataset_frames", "configs", "metrics", "rays", "train_data", "DeviceRayBatches", "importance_subsample_plan", "regular_subsample_plan", "Cfg", "to_cfg", "load_model_yaml", "epochs_to_iters", "LightfieldModel", "model_dict",
           "RenderLightfield", "render_chunked", "render_fn_dict", "Signature", "UnsupportedPipeline", "lower",
           "INRSystem", "fit"]
