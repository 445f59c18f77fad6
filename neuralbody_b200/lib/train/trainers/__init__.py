"""Drop-ins for the reference's `lib/train/trainers/` network wrappers."""
