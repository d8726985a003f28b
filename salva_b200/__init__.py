"""salva_b200 — H100-native SPH fluid-step engine behind salva3d's LiquidWorld::step surface.

Product code only: CUDA kernels + C ABI (csrc/, include/sph.h) and the host mirror of the reference
interface (liquid_world.py).  Nothing here imports the CPU oracle.
"""
from .liquid_world import (Akinci2013SurfaceTension, ArtificialViscosity, Becker2009Elasticity, Boundary,  # noqa: F401
                           DFSPHSolver, DFSPHViscosity, Fluid, He2014SurfaceTension, IISPHSolver, InteractionGroups, LiquidWorld, SphError,
                           WCSPHSurfaceTension, XSPHViscosity, StaticSampling, DynamicContactSampling, BODY_NONE, BODY_FIXED,
                           BODY_DYNAMIC, Cylinder, Cone, SurfaceAnisotropy, VorticityConfinement)
