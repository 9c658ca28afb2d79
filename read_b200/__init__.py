"""read_b200 — H100-native (sm_90a) implementation of READ's per-frame render hot path.

    points -> packed z-buffer pyramid -> descriptor feature pyramid -> gated-conv refinement net -> RGB

Host-side mirrors of the reference interfaces (same names / arguments / errors):
    read_b200.pcpr.forward            <- pcpr.forward            (MyRender/CloudProjection/pcpr_cuda.cpp)
    read_b200.myrender.MyRender       <- READ.gl.myrender.MyRender (src/READ/gl/myrender.py)
    read_b200.texture.PointTexture    <- READ.models.texture.PointTexture
    read_b200.compose.NetAndTexture   <- READ.models.compose.NetAndTexture
    read_b200.unet.UNet               <- READ.models.unet.UNet
    read_b200.pipeline.TexturePipeline<- READ.pipelines.ogl.TexturePipeline
All compute goes through the C-ABI library ``libread_b200.so`` (include/read_b200.h).  No CPU fallback.
"""
__version__ = "0.1.0"
