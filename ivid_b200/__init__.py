"""ivid_b200 — Hopper-native (H100, sm_90a) sampling hot path of JeffreyXiang/ivid.

Drop-in surface (same names as the reference packages `diffusion.backbones`, `diffusion.frameworks`,
`diffusion.samplers`, `rgbd_3d`):

    import ivid_b200.backbones as backbones      # AdmUnet2d
    import ivid_b200.frameworks as frameworks    # GaussianDiffusion, ClassifierFreeGuidance, InpaintCFG, SuperResCFG
    import ivid_b200.samplers as samplers        # DdpmSampler, DdimSampler
    import ivid_b200.rgbd_3d as rgbd_3d          # AggregationRenderer, utils.*

All compute goes through libivid_b200.so (C ABI in include/ivid_b200.h); there is no CPU fallback.
"""
__version__ = "0.1.0"
