"""objgan_b200 -- Hopper-native (H100, sm_90a) hot path of Obj-GAN's image_generation
training step.  See DESIGN.md.  Import as ``objgan_b200`` (shim package at repo root)."""
__version__ = "0.1.0"


def __getattr__(name):
    # GSampler is exported lazily: importing the package must not pull in torch and the model
    if name == "GSampler":
        from .sampler import GSampler
        return GSampler
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
