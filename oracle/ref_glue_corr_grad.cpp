// ORACLE glue (test infrastructure only): python bindings for the backward entries of the reference's correlation
// kernels (src/correlation_kernels.cu:157-185, src/altcorr_kernel.cu:321-356), compiled from the reference tree by
// oracle/build_ref_corr_grad.py into its own module, nslam_ref_corr_grad.  Mirrors src/droid.cpp:290-301, 315-327.
#include <torch/extension.h>
#include <vector>
std::vector<torch::Tensor> corr_index_cuda_backward(torch::Tensor volume, torch::Tensor coords, torch::Tensor corr_grad,
                                                    int radius);
std::vector<torch::Tensor> altcorr_cuda_backward(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor coords,
                                                 torch::Tensor corr_grad, int radius);
PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("corr_index_backward", &corr_index_cuda_backward);
  m.def("altcorr_backward", &altcorr_cuda_backward);
}
