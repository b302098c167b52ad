"""Drop-in for the original project's simple_knn extension (submodules/simple-knn): `from simple_knn._C import distCUDA2`."""
