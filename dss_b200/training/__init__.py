"""The training step next to the hot path (SURVEY.md 8(f)2): the projection / repulsion losses of
DSS/training/losses.py on top of the CUDA K-NN, and the image loss of Trainer.calc_dr_loss."""
from .losses import (BaseLoss, IouLoss, L1Loss, L2Loss, ProjectionLoss, RepulsionLoss, SurfaceLoss,  # noqa: F401
                     image_loss, image_loss_torch)
