"""Drop-in ``simple_knn`` package: the reference imports ``from simple_knn._C import distCUDA2``
(scene/gaussian_model.py:20) to set the initial Gaussian scales (:315-316).  Backed by the sm_90a kernels of
``rgs_knn.cu`` through the rasterizer's extension; no separate build or installation."""
