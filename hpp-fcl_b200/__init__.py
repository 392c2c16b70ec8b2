"""hpp-fcl_b200 -- batched narrow-phase collision/distance engine for the NVIDIA H100.

Host-side mirror (Python) of the hpp-fcl query interface for the hot path
collide()/distance() -> ShapeShapeDistance -> GJK/EPA (+ OBBRSS BVH traversal),
on top of the C-ABI shared library built from csrc/ (include/hppfcl_b200.h).
There is no CPU fallback: every query runs hand-written sm_90a CUDA kernels and
raises if the extension or a GPU is missing.
"""
from . import _pod  # noqa: F401
from ._pod import *  # noqa: F401,F403
from .build import build_extension, library_path  # noqa: F401
from .engine import (  # noqa: F401
    Engine, EngineError, broadphase_config_distance_pairs, broadphase_config_pairs, broadphase_cross_pairs,
    broadphase_pairs, broadphase_sweep_pairs, build_bvh_obbrss, load_library, robot_desc,
)
from .api import (  # noqa: F401
    BVHModelOBB, BVHModelOBBRSS, Box, Capsule, CollisionRequest, CollisionResult, Cone, Contact, Convex, Cylinder,
    DistanceRequest, DistanceResult, Ellipsoid, Halfspace, Plane, Sphere, Transform3f, TriangleP,
    collide, distance, ComputeCollision, ComputeDistance, BatchQuery,
    AABB, CollisionObject, CollisionCallBackCollect, DynamicAABBTreeCollisionManager, ResidentEnvironment,
    RobotModel, RobotSamples,
)
