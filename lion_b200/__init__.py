"""lion_b200 -- a from-scratch, H100-native (sm_90a) implementation of the sampling hot path
of nv-tlabs/LION: hand-written CUDA kernels behind a C ABI (include/lion_b200.h), with a
host-side mirror of the reference's Python interface for that path:

    lion_b200.third_party.pvcnn.functional      the 7 point/voxel operators
    lion_b200.models.pvcnn2_ada / .latent_points_ada / .latent_points_ada_localprior
    lion_b200.models.score_sde.resnet / .vae_adain
    lion_b200.utils.diffusion_pvd               DiffusionDiscretized (DDPM + DDIM loops)
    lion_b200.models.lion                       LION (demo wrapper; diffusers-style scheduler restated)
    lion_b200.third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D   Chamfer NN (metrics)
    lion_b200.third_party.PyTorchEMD.emd_nograd / .emd                       approximate EMD (metrics)
    lion_b200.utils.evaluation_metrics_fast     pairwise CD / EMD matrices, MMD / COV / 1-NNA and JSD scores
    lion_b200.utils.eval_helper / .data_helper  compute_score of a sample file, normalize_point_clouds
    lion_b200.trainers.train_2prior             generate_samples_vada_2prior (DDPM, DDIM and ODE routes)
    lion_b200.trainers.train_prior              Trainer.sample / Trainer.eval_sample (sampling-side Trainer)
    lion_b200.models.pvcnn2 / .shapelatent_modules / .distributions          VAE encoder path (non-Ada blocks)
    lion_b200.utils.diffusion_continuous        VPSDE, probability-flow ODE sampler and encoder (compute_ode_nll)
    lion_b200.trainers.interpolate_latent       latent interpolation by ODE sampling (script/interpolate.sh)
    lion_b200.trainers.encode_interp_interp     interpolation between encoded shapes (script/interpolate_posterior.sh)

`lion_b200.install()` registers these under the reference's own import paths (`models.*`,
`utils.diffusion_pvd`, `trainers.train_2prior`, `third_party.pvcnn.functional`) so that
reference entry points (demo.py, train_dist.py --eval_generation) pick them up unchanged.
"""
import importlib
import sys

__version__ = "0.1.0"

_ALIASES = {
    "third_party.pvcnn.functional": "lion_b200.third_party.pvcnn.functional",
    "third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D":
        "lion_b200.third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D",
    "third_party.PyTorchEMD.emd_nograd": "lion_b200.third_party.PyTorchEMD.emd_nograd",
    "third_party.PyTorchEMD.emd": "lion_b200.third_party.PyTorchEMD.emd",
    "models.adagn": "lion_b200.models.adagn",
    "models.dense": "lion_b200.models.dense",
    "models.pvcnn2_ada": "lion_b200.models.pvcnn2_ada",
    "models.pvcnn2": "lion_b200.models.pvcnn2",
    "models.shapelatent_modules": "lion_b200.models.shapelatent_modules",
    "models.distributions": "lion_b200.models.distributions",
    "models.latent_points_ada": "lion_b200.models.latent_points_ada",
    "models.latent_points_ada_localprior": "lion_b200.models.latent_points_ada_localprior",
    "models.score_sde.resnet": "lion_b200.models.score_sde.resnet",
    "models.vae_adain": "lion_b200.models.vae_adain",
    "models.lion": "lion_b200.models.lion",
    "utils.diffusion_pvd": "lion_b200.utils.diffusion_pvd",
    "utils.diffusion_continuous": "lion_b200.utils.diffusion_continuous",
    "trainers.train_2prior": "lion_b200.trainers.train_2prior",
    "trainers.interpolate_latent": "lion_b200.trainers.interpolate_latent",
    "trainers.encode_interp_interp": "lion_b200.trainers.encode_interp_interp",
}


def install():
    """Make the reference's import paths resolve to this package (drop-in for the hot path)."""
    for ref_name, ours in _ALIASES.items():
        sys.modules[ref_name] = importlib.import_module(ours)
