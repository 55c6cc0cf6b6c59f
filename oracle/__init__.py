"""CPU oracle for the CaTGrasp hot path -- TEST INFRASTRUCTURE ONLY.

Nothing under ``catgrasp_b200/`` may import this package.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl reference``
legs use it, as the checker and as the timed CPU baseline -- never as the product.

Pinning status (DESIGN.md section "Oracle"):
  * pointnet_ref.py, pn2_ref.py : PINNED against the reference's own pointnet2.py executed in the
    authoring container (tests/golden/make_golden.py -> tests/golden/*.npz).
  * transforms_ref.py, aligning_ref.py : PINNED against the reference's own predicter.py / dataset_grasp.py /
    dataset_nunocs.py / augmentations.py / aligning.py / Utils.load_model executed in the authoring container with
    the absent third-party imports stubbed (tests/golden/make_golden_hostpath.py -> tests/golden/host_*.npz).
  * sdf_ref.py                  : PINNED against the reference's meshpy Sdf3D lookups / SdfFile reader executed here
    (tests/golden/make_golden_sdf.py -> sdf_lookup.npz).
  * affordance_ref.py           : PINNED against the reference's compute_grasp_affordance_worker / get_finger_contact_area
    (tests/golden/make_golden_affordance.py -> affordance.npz).
  * fcl_semantic_ref.py         : NOT a pin -- a restatement of the FCL/octomap mesh-vs-voxel semantic used only to measure
    the agreement rate of the SDF predicate with it (tests/test_fcl_semantic_agreement.py).
  * cone_ref.py                 : PINNED against poses recorded from the reference's PointConeGraspSampler.sample_grasps
    (tests/golden/make_golden_cone.py -> cone_poses.npz).
  * filter_ref.c, occupancy_ref.c : pose logic / control flow PINNED against the reference's own my_cpp/common.cpp
    compiled by oracle/build_ref.py into oracle/_ref (bit-identical survivor sets / occupied samples,
    tests/golden/make_golden_mycpp.py -> tests/golden/mycpp_*.npz).  The FCL / octomap boundary cannot be built
    here (libraries absent, versions unpinned) -> that part is parity UNPINNED; both sides use the gripper-SDF
    predicate of meshpy/sdf.py and a restatement of the octomap calls instead (oracle/ref_shim/).
  * filter64.py                 : float64 statement of the filter's predicate on sdf_ref.py's lookups, with a rigorous
    bound on the float32 pipeline; checks filter_ref.c and the kernel on every verdict the bound decides
    (tests/test_filter_ref.py, tests/test_filter_kernel.py).
  * ransac64.py                 : one RANSAC hypothesis in high precision (cv2's 4-point affine, gate margins, a bound on
    the kernel's T, the inlier count as an interval); pinned to cv2 via aligning_ref._hypothesis (tests/test_ransac_ref.py).
"""
