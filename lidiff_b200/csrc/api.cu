// Dispatch of lb2_spconv_forward to the CUDA-core (spconv_ffma.cu) or wgmma (spconv_tc.cu) variant.
#include "common.cuh"

int lb2_spconv_ffma_launch(Lb2Handle* h, cudaStream_t s, const lb2_conv_desc* d);
int lb2_spconv_tc_launch(Lb2Handle* h, cudaStream_t s, const lb2_conv_desc* d);
bool lb2_spconv_tc_supported(const lb2_conv_desc* d);

extern "C" int lb2_spconv_forward(void* handle, void* stream, const lb2_conv_desc* d, int algo) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && d, "spconv_forward null");
    LB2_REQUIRE(h, d->npass == 1 || d->npass == 2, "npass must be 1 or 2");
    LB2_REQUIRE(h, d->c1 > 0 && d->c2 >= 0 && d->cout > 0 && d->kvol > 0 && d->mout_cap > 0, "shape");
    LB2_REQUIRE(h, d->weight != nullptr, "weight");
    LB2_REQUIRE(h, (d->scale == nullptr) == (d->shift == nullptr), "scale/shift must come together");
    LB2_REQUIRE(h, d->nbr != nullptr || d->kvol == 1, "identity map only for kvol == 1");
    LB2_REQUIRE(h, d->nbr == nullptr || d->nbr_stride >= d->mout_cap, "nbr_stride");
    bool have_f32 = true;                                  // every pass has its inputs as fp32 tensors (CUDA-core variant needs them)
    for (int p = 0; p < d->npass; ++p) {
        const lb2_conv_io& io = d->io[p];
        const bool f = io.in1 && (d->c2 == 0 || io.in2), hh = io.in1_h && (d->c2 == 0 || io.in2_h);
        LB2_REQUIRE(h, f || hh, "in1 / in2 (fp32 tensors or their split companions)");
        LB2_REQUIRE(h, d->c2 > 0 || (io.in2 == nullptr && io.in2_h == nullptr), "in2 / c2 mismatch");
        LB2_REQUIRE(h, !hh || (d->c1 % 8 == 0 && d->c2 % 8 == 0), "split companions need channel counts that are multiples of 8");
        LB2_REQUIRE(h, io.out || io.out_gated || io.out_h || io.out_gated_h, "no output");
        have_f32 = have_f32 && f;
    }
    LB2_REQUIRE(h, d->c2 == 0 || d->c1 % 16 == 0, "c1 must be a multiple of 16 when in2 is given");
    cudaStream_t s = (cudaStream_t)stream;
    if (d->k1 > 0) {                                       // offset ranges: the tensor-core variant only
        if (algo == LB2_ALGO_FFMA || !d->weight_packed || !lb2_spconv_tc_supported(d))
            return lb2_fail(h, LB2_ERR_UNSUP, "an offset range needs the tensor-core variant%s", "");
        return lb2_spconv_tc_launch(h, s, d);
    }
    if (algo == LB2_ALGO_TC || algo == LB2_ALGO_TC_TILE) {
        if (!d->weight_packed || !lb2_spconv_tc_supported(d))
            return lb2_fail(h, LB2_ERR_UNSUP, "tensor-core variant does not support this layer%s", "");
        return lb2_spconv_tc_launch(h, s, d);
    }
    if (algo == LB2_ALGO_AUTO && d->weight_packed && lb2_spconv_tc_supported(d)) return lb2_spconv_tc_launch(h, s, d);
    if (!have_f32) return lb2_fail(h, LB2_ERR_UNSUP, "companion-only inputs need a tensor-core variant that takes this layer%s", "");
    return lb2_spconv_ffma_launch(h, s, d);
}
