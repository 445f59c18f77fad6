"""Host-side drop-ins for the reference's `lib/train/` modules."""
