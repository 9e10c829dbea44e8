// shencoder.cu -- real spherical-harmonics direction encoding, degree 1..8, for sm_90a.
//
// Replaces the native layer behind the reference's `sh_encode` / `SHEncoder`
// (reference: shencoder/src/shencoder.cu:28-439).  The reference spells out 64 polynomials and
// their 192 partial derivatives; here the same polynomials are generated from the factorisation
//     Y_l^{+m} = K_lm * Q_l^m(z) * Re (x+iy)^m,   Y_l^{-m} = K_lm * Q_l^m(z) * Im (x+iy)^m
// with Q_l^m = d^m/dz^m P_l(z) (Legendre, no Condon-Shortley factor; the phase (-1)^m and the
// sqrt(2) live in K_lm) evaluated by the standard three-term recurrence.  Because the reference's
// polynomials are exactly this product form (z-only Legendre factor times an (x,y)-only
// azimuthal factor, also off the unit sphere), the analytic derivatives agree too:
//     d/dx: m * Q * Re/Im (x+iy)^(m-1),   d/dy: -/+ m * Q * Im/Re (x+iy)^(m-1),   d/dz: Q_l^{m+1} * (..)
// Output index = l*l + l + m, dy_dx layout [B, 3, degree^2] (dx block, dy block, dz block).
#include "n2m_common.cuh"

namespace n2m {
namespace {

// K_lm = sqrt((2l+1)/(4 pi) * (l-m)!/(l+m)!) * (m > 0 ? sqrt(2) * (-1)^m : 1), generated in double.
__device__ const float kShNorm[8][8] = {
    {0.28209479177387814f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f},
    {0.48860251190291992f, -0.48860251190291998f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f},
    {0.63078313050504009f, -0.36418281019735976f, 0.18209140509867988f, 0.f, 0.f, 0.f, 0.f, 0.f},
    {0.7463526651802308f, -0.3046971996429772f, 0.096353714754685155f, -0.039336239328442907f, 0.f, 0.f, 0.f, 0.f},
    {0.84628437532163447f, -0.26761861742291571f, 0.063078313050504001f, -0.016858388283618388f, 0.0059603403376112026f, 0.f, 0.f, 0.f},
    {0.9356025796273888f, -0.24157154730437169f, 0.045652731285460234f, -0.0093188247511476283f, 0.0021964680580751762f, -0.00069458418713245519f, 0.f, 0.f},
    {1.0171072362820548f, -0.22195099524523101f, 0.03509353369580661f, -0.0058489222826344353f, 0.0010678622237644956f, -0.00022766899107568562f, 6.5722376641838803e-05f, 0.f},
    {1.0925484305920792f, -0.20647224590289676f, 0.028097313806030647f, -0.0039735602250741348f, 0.00059903674311141165f, -9.9839457185235285e-05f, 1.9580128477462541e-05f, -5.233009453691466e-06f},
};

template <int DEG, bool WITH_GRAD>
__global__ void __launch_bounds__(256)
k_sh_fwd(const float* __restrict__ inputs, float* __restrict__ outputs, uint32_t B, uint32_t D, float* __restrict__ dy_dx) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    constexpr int C2 = DEG * DEG;
    const float x = inputs[(size_t)b * D], y = inputs[(size_t)b * D + 1], z = inputs[(size_t)b * D + 2];
    float* out = outputs + (size_t)b * C2;
    float* gx = WITH_GRAD ? dy_dx + (size_t)b * D * C2 : nullptr;
    float* gy = WITH_GRAD ? gx + C2 : nullptr;
    float* gz = WITH_GRAD ? gy + C2 : nullptr;

    // azimuthal factors A_m = Re (x+iy)^m, B_m = Im (x+iy)^m
    float A[DEG], Bm[DEG];
    A[0] = 1.f; Bm[0] = 0.f;
#pragma unroll
    for (int m = 1; m < DEG; ++m) {
        A[m] = x * A[m - 1] - y * Bm[m - 1];
        Bm[m] = x * Bm[m - 1] + y * A[m - 1];
    }

    // Q[m][l] for l = m..DEG-1, plus one extra order for the z-derivative (Q_l^{m+1} = dQ_l^m/dz)
    float Q[DEG + 1][DEG];
#pragma unroll
    for (int m = 0; m <= DEG; ++m) {
        float dfact = 1.f;                      // (2m-1)!!
#pragma unroll
        for (int k = 1; k <= m; ++k) dfact *= (float)(2 * k - 1);
#pragma unroll
        for (int l = 0; l < DEG; ++l) {
            if (l < m) Q[m][l] = 0.f;
            else if (l == m) Q[m][l] = dfact;
            else if (l == m + 1) Q[m][l] = (float)(2 * m + 1) * z * Q[m][m];
            else Q[m][l] = ((float)(2 * l - 1) * z * Q[m][l - 1] - (float)(l + m - 1) * Q[m][l - 2]) / (float)(l - m);
        }
    }

#pragma unroll
    for (int l = 0; l < DEG; ++l) {
#pragma unroll
        for (int m = 0; m <= l; ++m) {
            const float k = kShNorm[l][m];
            const float q = k * Q[m][l];
            const int ip = l * l + l + m, in = l * l + l - m;
            out[ip] = q * A[m];
            if (m > 0) out[in] = q * Bm[m];
            if (WITH_GRAD) {
                const float qz = k * Q[m + 1][l];
                const float am1 = m > 0 ? A[m - 1] : 0.f, bm1 = m > 0 ? Bm[m - 1] : 0.f;
                gx[ip] = q * ((float)m * am1);
                gy[ip] = q * (-(float)m * bm1);
                gz[ip] = qz * A[m];
                if (m > 0) {
                    gx[in] = q * ((float)m * bm1);
                    gy[in] = q * ((float)m * am1);
                    gz[in] = qz * Bm[m];
                }
            }
        }
    }
}

// grad_inputs[b, d] += sum_ch grad[b, ch] * dy_dx[b, d, ch]   (shencoder.cu:359-382)
__global__ void __launch_bounds__(256)
k_sh_bwd(const float* __restrict__ grad, uint32_t B, uint32_t D, uint32_t C2, const float* __restrict__ dy_dx,
         float* __restrict__ grad_inputs) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t b = t / D;
    if (b >= B) return;
    const uint32_t d = t - b * D;
    const float* g = grad + (size_t)b * C2;
    const float* dd = dy_dx + ((size_t)b * D + d) * C2;
    float acc = grad_inputs[t];
    for (uint32_t ch = 0; ch < C2; ++ch) acc += g[ch] * dd[ch];
    grad_inputs[t] = acc;
}

template <int DEG>
int launch_sh(const float* inputs, float* outputs, uint32_t B, uint32_t D, float* dy_dx, cudaStream_t st) {
    if (dy_dx) k_sh_fwd<DEG, true><<<div_up(B, 256u), 256, 0, st>>>(inputs, outputs, B, D, dy_dx);
    else k_sh_fwd<DEG, false><<<div_up(B, 256u), 256, 0, st>>>(inputs, outputs, B, D, nullptr);
    return check_launch("sh_encode_forward");
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_sh_encode_forward(const float* inputs, float* outputs, uint32_t B, uint32_t D, uint32_t degree, float* dy_dx,
                          n2m_stream_t stream) {
    if (B == 0) return 0;
    N2M_REQUIRE(inputs && outputs, "sh_encode_forward", "null pointer");
    N2M_REQUIRE(D == 3, "sh_encode_forward", "SH encoder only support input dim == 3");
    cudaStream_t st = as_stream(stream);
    switch (degree) {
        case 1: return launch_sh<1>(inputs, outputs, B, D, dy_dx, st);
        case 2: return launch_sh<2>(inputs, outputs, B, D, dy_dx, st);
        case 3: return launch_sh<3>(inputs, outputs, B, D, dy_dx, st);
        case 4: return launch_sh<4>(inputs, outputs, B, D, dy_dx, st);
        case 5: return launch_sh<5>(inputs, outputs, B, D, dy_dx, st);
        case 6: return launch_sh<6>(inputs, outputs, B, D, dy_dx, st);
        case 7: return launch_sh<7>(inputs, outputs, B, D, dy_dx, st);
        case 8: return launch_sh<8>(inputs, outputs, B, D, dy_dx, st);
    }
    return fail("sh_encode_forward", "SH encoder only supports degree in [1, 8]");
}

int n2m_sh_encode_backward(const float* grad, const float* inputs, uint32_t B, uint32_t D, uint32_t degree,
                           const float* dy_dx, float* grad_inputs, n2m_stream_t stream) {
    (void)inputs;
    if (B == 0) return 0;
    N2M_REQUIRE(grad && dy_dx && grad_inputs, "sh_encode_backward", "null pointer");
    N2M_REQUIRE(D == 3, "sh_encode_backward", "SH encoder only support input dim == 3");
    N2M_REQUIRE(degree >= 1 && degree <= 8, "sh_encode_backward", "SH encoder only supports degree in [1, 8]");
    k_sh_bwd<<<div_up(B * D, 256u), 256, 0, as_stream(stream)>>>(grad, B, D, degree * degree, dy_dx, grad_inputs);
    return check_launch("sh_encode_backward");
}

}  // extern "C"
