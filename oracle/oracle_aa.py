"""The C oracle (oracle/oracle_c.py, oracle/sgn_oracle.c, used unchanged) in the antialiased rasterize mode.  TEST
INFRASTRUCTURE -- never imported by the product.

The mode changes one input of the blend -- the opacity of a visible Gaussian becomes sigmoid(logit) * comp -- and adds one
path to the backward -- comp's own gradient through cov2d.  Both come from the float64 statement
(oracle/project_aa_ref64.py):
  * ``project``: the C oracle's projection with ``opac`` = float32(sigmoid * comp) on its visible rows (radii > 0), 0
    elsewhere; the blend, the fragile-pixel flags and the per-entry touch test then run on that opacity, as the kernels do;
  * ``project_bwd``: the blend's opacity cotangent v (w.r.t. sigmoid * comp) enters the C projection backward as v * comp
    (the logit's share: v comp s (1 - s)), and the float64 gradient of sum(comp * v * s) w.r.t. means, scales and quats is
    added to its geometry gradients.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from oracle import oracle_c
from oracle import project_aa_ref64 as aa
from oracle import project_ref64 as ref


class AntialiasedOracle(oracle_c.Oracle):
    def __init__(self, frame, sh_degree: int = 3, sh_degree_to_use: Optional[int] = None, block_width: int = 16,
                 clip_thresh: float = 0.01, **kw):
        super().__init__(frame, sh_degree, sh_degree_to_use, block_width, clip_thresh, **kw)
        self.st = ref.Settings(sh_degree=sh_degree, sh_degree_to_use=sh_degree_to_use, block_width=block_width,
                               clip_thresh=clip_thresh)
        self._comp = None

    def comp(self) -> np.ndarray:
        """float64 comp of every row (unmasked; the caller selects the visible ones)."""
        if self._comp is None:
            leaves = [{k: getattr(sg.params, k).detach().cpu().double() for k in ("means", "scales", "quats")}
                      for sg in self.frame.segments]
            pr = aa._geometry(self.frame, leaves, self.st, torch.float64)
            self._comp = aa.compensation(pr["a"], pr["b"], pr["c"]).numpy()
        return self._comp

    def sigmoid(self) -> np.ndarray:
        logit = np.concatenate([sg.params.opacities.detach().cpu().double().numpy()[:, 0] for sg in self.frame.segments])
        return 1.0 / (1.0 + np.exp(-logit))

    def project(self):
        pr = super().project()
        vis = pr["radii"] > 0
        pr["opac"] = np.where(vis, pr["opac"].astype(np.float64) * self.comp(), 0.0).astype(np.float32)
        return pr

    def project_bwd(self, fw, v_xy, v_depth, v_conic, v_rgb, v_opac):
        vis = fw.radii > 0
        comp = np.where(vis, self.comp(), 0.0)
        v_opac = np.asarray(v_opac, np.float64)
        grads = super().project_bwd(fw, v_xy, v_depth, v_conic, v_rgb, (v_opac * comp).astype(np.float32))
        extra = aa.comp_param_grads(self.frame, self.st, np.where(vis & (comp > 0), v_opac * self.sigmoid(), 0.0))
        for g, e in zip(grads, extra):
            for k in ("means", "scales", "quats"):
                g[k] = (g[k].astype(np.float64) + e[k]).astype(np.float32)
        return grads
