"""Drop-in package name for the reference's import
    from simple_knn._C import distCUDA2
(scene/gaussian_model.py:20, games/flat_splatting/scene/flat_gaussian_model.py:19).  With `gaussian-mesh-splatting_b200/` on
sys.path, the reference's create_from_pcd runs on this library's exact three-nearest-neighbour kernel."""
