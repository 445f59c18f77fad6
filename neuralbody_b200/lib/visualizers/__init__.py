"""Host-side drop-ins for the reference's `lib/visualizers/` modules."""
