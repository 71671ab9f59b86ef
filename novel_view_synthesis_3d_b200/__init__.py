"""novel_view_synthesis_3d_b200 -- the X-UNet pose-conditional denoiser hot path of
shiveshkhaitan/novel_view_synthesis_3d, rebuilt H100-native (hand-written sm_90a CUDA behind a C-ABI)."""
from .xunet import XUNet, XUNetConfig, SMALL, FULL_3DIM, ParamTree, Engine
from .train import (TrainState, Adam, AdamState, create_train_state, create_sample_data, apply_model, update_model,
                    TrainStep)
from . import checkpoint, consistency, distill, lift, metrics, pose, posthoc, sampling, srn_data
from .consistency import Field, consistency_score, fit_field
from .distill import ConsistencyTeacher, Teacher, create_distill_state
from .pose import PoseEstimator, PoseResult, rotation_error_deg
from .lift import FieldLifter, LiftResult, estimate_up, elevation_range
from .diffusion import ForwardDiffusion
from .srn_data import DeviceScenes
from .metrics import image_metrics
from .sampling import Sampler, Schedule, consistency_grid, cosine_beta_schedule, distill_grid, logsnr_schedule_cosine

__all__ = ['XUNet', 'XUNetConfig', 'SMALL', 'FULL_3DIM', 'ParamTree', 'Engine', 'TrainState', 'Adam', 'AdamState',
           'create_train_state', 'create_sample_data', 'apply_model', 'update_model', 'TrainStep', 'Sampler',
           'Schedule', 'cosine_beta_schedule', 'logsnr_schedule_cosine', 'checkpoint', 'ForwardDiffusion', 'metrics',
           'image_metrics', 'DeviceScenes', 'distill', 'Teacher', 'create_distill_state', 'distill_grid',
           'consistency', 'Field', 'fit_field', 'consistency_score', 'pose', 'PoseEstimator', 'PoseResult',
           'rotation_error_deg', 'lift', 'FieldLifter', 'LiftResult', 'estimate_up', 'elevation_range',
           'ConsistencyTeacher', 'consistency_grid', 'posthoc']
