"""vlfb -- H100-native engine behind the reference's lib/models builder API.

`cnn.CNNModelHelper` / `workspace` stand in for the caffe2.python modules the reference
imports (lib/models/model_builder_video.py:27-34); `kernels` binds libvlfb.so (C ABI in
include/vlfb.h); `executor` lowers recorded nets onto the sm_90a kernels; `dist` is the
one-process-per-GPU data-parallel plumbing (NCCL all-reduce of gradients).
"""
