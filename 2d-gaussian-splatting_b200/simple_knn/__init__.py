"""Drop-in for the reference's `simple_knn` extension (submodules/simple-knn): `from simple_knn._C import distCUDA2`
(/root/reference/scene/gaussian_model.py:20) resolves here, backed by the sm_90a library of this project."""
