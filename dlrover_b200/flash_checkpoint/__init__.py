"""H100-native Flash Checkpoint: the trainer-side API of
dlrover.trainer.torch.flash_checkpoint re-implemented over libflashckpt."""
