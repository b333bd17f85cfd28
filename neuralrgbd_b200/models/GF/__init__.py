"""Mirrors of the reference's models/GF package: GuidedFilter and BoxFilter on libnrgbd kernels, with autograd."""
