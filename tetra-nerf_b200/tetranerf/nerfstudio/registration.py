"""nerfstudio method registration: `tetra-nerf` (128+128 samples, biased sampler, gradient scaling) and
`tetra-nerf-original` (256+256, uniform) -- reference tetranerf/nerfstudio/registration.py:20-67.
Control plane, outside the hot-path scope; requires nerfstudio."""
import dataclasses
from functools import partial

from nerfstudio.data.datamanagers.base_datamanager import VanillaDataManagerConfig
from nerfstudio.engine.optimizers import RAdamOptimizerConfig
from nerfstudio.engine.schedulers import ExponentialDecaySchedulerConfig
from nerfstudio.engine.trainer import TrainerConfig
from nerfstudio.pipelines.base_pipeline import VanillaPipelineConfig
from nerfstudio.plugins.types import MethodSpecification

try:
    from nerfstudio.data.dataparsers.colmap_dataparser import ColmapDataParserConfig

    _DataParser = partial(ColmapDataParserConfig, load_3D_points=True)
except ImportError:  # older nerfstudio
    from nerfstudio.data.dataparsers.minimal_dataparser import MinimalDataParserConfig as _DataParser

from .model import TetrahedraNerf, TetrahedraNerfConfig
from .pipeline import TetrahedraNerfPipeline


def _trainer(name: str, model: TetrahedraNerfConfig) -> TrainerConfig:
    return TrainerConfig(
        method_name=name,
        pipeline=VanillaPipelineConfig(
            _target=TetrahedraNerfPipeline,
            datamanager=VanillaDataManagerConfig(dataparser=_DataParser(), train_num_rays_per_batch=4096, eval_num_rays_per_batch=4096),
            model=model,
        ),
        max_num_iterations=300000, steps_per_save=25000, steps_per_eval_batch=1000, steps_per_eval_image=2000, steps_per_eval_all_images=50000,
        optimizers={"fields": {"optimizer": RAdamOptimizerConfig(lr=0.001),
                               "scheduler": ExponentialDecaySchedulerConfig(lr_final=0.0001, max_steps=300_000)},
                    # the param group of TetrahedraNerfConfig.optimize_vertices; nerfstudio's Optimizers builds one optimizer per param
                    # group the model returns, so this entry is inert while the option is off.  The rate is a placeholder, not tuned.
                    "vertices": {"optimizer": RAdamOptimizerConfig(lr=1e-5),
                                 "scheduler": ExponentialDecaySchedulerConfig(lr_final=1e-6, max_steps=300_000)}},
    )


tetranerf_original_config = _trainer("tetra-nerf-original", TetrahedraNerfConfig(_target=TetrahedraNerf))
tetranerf_config = _trainer("tetra-nerf", dataclasses.replace(TetrahedraNerfConfig(_target=TetrahedraNerf), num_samples=128, num_fine_samples=128,
                                                              use_biased_sampler=True, use_gradient_scaling=True))
tetranerf_original = MethodSpecification(config=tetranerf_original_config, description="Official implementation of Tetra-NeRF paper")
tetranerf = MethodSpecification(config=tetranerf_config, description="Newer version of Tetra-NeRF with better performance")
