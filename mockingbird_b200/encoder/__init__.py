"""Speaker encoder on the H100 path (reference: models/encoder)."""
