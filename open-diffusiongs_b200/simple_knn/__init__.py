"""Drop-in `simple_knn` package backed by libdgs_b200.so (sm_90a): `from simple_knn._C import distCUDA2`, as 3DGS-family
code imports it from the reference's submodules/simple-knn to initialise Gaussian scales."""
