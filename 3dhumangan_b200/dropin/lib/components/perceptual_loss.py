import importlib as _il

VGGPerceptualLoss = _il.import_module("3dhumangan_b200.perceptual").VGGPerceptualLoss
