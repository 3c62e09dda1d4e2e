"""Configuration objects for the sampling path.

The modules read the same attribute paths as the reference (`cfg.ddpm.num_steps`,
`cfg.latent_pts.style_dim`, `cfg.sde.embedding_dim`, ...) so a yacs CfgNode built by the
reference's `default_config.py` + `config/*_prior_cfg.yml` works unchanged; this file only
provides the same tree without the reference installed (values: config/airplane_prior_cfg.yml,
identical for chair/car except `sde.dropout`, SURVEY.md 8d).
"""
import copy


class Cfg(dict):
    """dict with attribute access (a minimal stand-in for yacs.CfgNode)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v

    def clone(self):
        return copy.deepcopy(self)

    def merge_from_list(self, opts):
        assert len(opts) % 2 == 0
        for k, v in zip(opts[0::2], opts[1::2]):
            node = self
            parts = k.split(".")
            for p in parts[:-1]:
                node = node[p]
            node[parts[-1]] = v
        return self


def _wrap(d):
    return Cfg({k: _wrap(v) if isinstance(v, dict) else v for k, v in d.items()})


_DEFAULT = {
    "ddpm": {"num_steps": 1000, "beta_1": 1e-4, "beta_T": 0.02, "sched_mode": "linear", "time_dim": 64,
             "input_dim": 3, "dropout": 0.1, "p2_gamma": 1.0, "p2_k": 1.0, "use_p2_weight": 0,
             "model_var_type": "fixedlarge"},
    "latent_pts": {"style_dim": 128, "ada_mlp_init_scale": 0.1, "skip_weight": 0.01, "pts_sigma_offset": 0.0,
                   "style_mlp": "", "style_prior": "models.score_sde.resnet.PriorSEDrop",
                   "style_encoder": "models.shapelatent_modules.PointNetPlusEncoder"},
    "shapelatent": {"latent_dim": 1, "decoder_type": "models.latent_points_ada.LatentPointDecPVC",
                    "encoder_type": "models.latent_points_ada.PointTransPVC", "kl_weight": 0.5,
                    "log_sigma_offset": 6.0},
    "sde": {"mixed_prediction": False, "mixing_logit_init": -6, "embedding_scale": 1.0, "embedding_dim": 128,
            "embedding_type": "positional", "num_channels_dae": 2048, "num_cell_per_scale_dae": 8,
            "num_scales_dae": 2, "dropout": 0.2, "learn_mixing_logit": 1, "ode_sample": 0, "sde_type": "vpsde", "sigma2_0": 0.0,
            "sigma2_min": 1e-4, "sigma2_max": 0.99, "beta_start": 0.1, "beta_end": 20.0, "time_eps": 0.01, "ode_eps": 1e-5,
            "train_ode_solver_tol": 1e-5, "autocast_train": False,
            "prior_model": "models.latent_points_ada_localprior.PVCNN2Prior"},
    "clipforge": {"enable": 0, "feat_dim": 512},
    "data": {"tr_max_sample_points": 2048, "cond_on_cat": 0, "batch_size_test": 10},
    "eval": {"need_denoise": 0},
    "trainer": {"seed": 1},
    "num_ref": 0,
}


def default_prior_cfg(clip=False, num_steps=None):
    cfg = _wrap(copy.deepcopy(_DEFAULT))
    if clip:
        cfg.clipforge.enable = 1
        cfg.latent_pts.style_prior = "models.score_sde.resnet.PriorSEClip"
    if num_steps is not None:
        cfg.ddpm.num_steps = num_steps
    return cfg


def load_yaml(path):
    """Read a reference-style YAML (e.g. config/airplane_prior_cfg.yml) over the defaults."""
    import yaml
    cfg = default_prior_cfg()
    with open(path) as f:
        user = yaml.safe_load(f)

    def merge(dst, src):
        for k, v in src.items():
            if isinstance(v, dict) and isinstance(dst.get(k), dict):
                merge(dst[k], v)
            else:
                dst[k] = _wrap(v) if isinstance(v, dict) else v
    merge(cfg, user)
    return cfg
