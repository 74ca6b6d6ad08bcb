// bsdf.cuh -- device-side PBR BSDF (Lambert / Frostbite diffuse + GGX specular) and the
// hand-derived adjoints.  Same math as the reference's two twins:
//   render/optixutils/c_src/bsdf.h:21-275      (in-kernel, demodulated diffuse, direction wi)
//   render/renderutils/c_src/bsdf.cu:17-377    (stand-alone ops, kd-modulated, light position)
// written for sm_90a: everything stays in registers, FMA contraction allowed (this is NOT on the
// sampling decision path), pow(x,5)/pow(x,3) expanded into multiplies, 1/pi folded into constants.
//
// Conditioning note: the GGX NDF denominator d = (c*a2 - c)*c + 1 cancels catastrophically at the
// specular peak (c -> 1, small roughness): in fp32 its relative rounding noise reaches ~1e-3, and the
// adjoint (~1/d^3) amplifies it further.  That noise is inherent to the reference's formula; to keep
// parity testable the half vector, n.h, the gate cosines and every expression containing d are
// evaluated with exact.cuh arithmetic in the oracle's operation order, so both sides carry the SAME
// rounding.  Everything else (Fresnel, masking, products, adjoint chains) is well conditioned and
// uses contracted fast math.
#pragma once
#include "common.cuh"
#include "exact.cuh"

#define MCS_SPEC_EPS 1e-4f
#define MCS_PI 3.14159265358979323846f
#define MCS_INV_PI 0.31830988618379067154f

// v / |v| with IEEE sqrt and divisions in the reference's order (math_utils.h:135-139)
__device__ __forceinline__ f3 safe_normalize(f3 v) { return toF3(xnormalize(X3(v))); }
__device__ __forceinline__ float dot_exact(f3 a, f3 b) { return xdot(X3(a), X3(b)).v; }
// adjoint of v / |v|   (math_utils.h:141-152)
__device__ __forceinline__ void bwd_safe_normalize(f3 v, f3 &d_v, f3 d_out)
{
    float l2 = dot(v, v);
    if (l2 > 0.0f) {
        float inv = rsqrtf(l2);
        float fac = inv * inv * inv;               // 1 / |v|^3
        d_v.x += (d_out.x * (v.y * v.y + v.z * v.z) - d_out.y * (v.x * v.y) - d_out.z * (v.x * v.z)) * fac;
        d_v.y += (d_out.y * (v.x * v.x + v.z * v.z) - d_out.x * (v.y * v.x) - d_out.z * (v.y * v.z)) * fac;
        d_v.z += (d_out.z * (v.x * v.x + v.y * v.y) - d_out.x * (v.z * v.x) - d_out.y * (v.z * v.y)) * fac;
    }
}
__device__ __forceinline__ void bwd_dot(f3 a, f3 b, f3 &d_a, f3 &d_b, float d_out)
{
    d_a += b * d_out;
    d_b += a * d_out;
}
__device__ __forceinline__ void bwd_cross(f3 a, f3 b, f3 &d_a, f3 &d_b, f3 d_out)
{
    d_a.x += d_out.z * b.y - d_out.y * b.z;
    d_a.y += d_out.x * b.z - d_out.z * b.x;
    d_a.z += d_out.y * b.x - d_out.x * b.y;
    d_b.x += d_out.y * a.z - d_out.z * a.y;
    d_b.y += d_out.z * a.x - d_out.x * a.z;
    d_b.z += d_out.x * a.y - d_out.y * a.x;
}
__device__ __forceinline__ float luminance(f3 c) { return dot(c, F3(0.2126f, 0.7152f, 0.0722f)); }
__device__ __forceinline__ float pow5f(float x) { float x2 = x * x; return x2 * x2 * x; }

// ---- Lambert (bsdf.h:21-30) -----------------------------------------------------------------
__device__ __forceinline__ float fwd_lambert(f3 nrm, f3 wi) { return fmaxf(dot(nrm, wi) * MCS_INV_PI, 0.0f); }
__device__ __forceinline__ void bwd_lambert(f3 nrm, f3 wi, f3 &d_nrm, f3 &d_wi, float d_out)
{
    if (dot(nrm, wi) > 0.0f) bwd_dot(nrm, wi, d_nrm, d_wi, d_out * MCS_INV_PI);
}

// ---- Schlick Fresnel (bsdf.h:35-71) ---------------------------------------------------------
__device__ __forceinline__ float schlick_scale(float cosTheta)
{
    float c = clampf(cosTheta, MCS_SPEC_EPS, 1.0f - MCS_SPEC_EPS);
    return pow5f(1.0f - c);
}
__device__ __forceinline__ float fwd_fresnel1(float f0, float f90, float cosTheta)
{
    float s = schlick_scale(cosTheta);
    return f0 * (1.0f - s) + f90 * s;
}
__device__ __forceinline__ void bwd_fresnel1(float f0, float f90, float cosTheta, float &d_f0, float &d_f90, float &d_cos, float d_out)
{
    float s = schlick_scale(cosTheta);
    d_f0 += d_out * (1.0f - s);
    d_f90 += d_out * s;
    if (cosTheta >= MCS_SPEC_EPS && cosTheta < 1.0f - MCS_SPEC_EPS) {
        float o = 1.0f - cosTheta, o2 = o * o;
        d_cos += d_out * (f90 - f0) * -5.0f * (o2 * o2);
    }
}
__device__ __forceinline__ f3 fwd_fresnel3(f3 f0, f3 f90, float cosTheta)
{
    float s = schlick_scale(cosTheta);
    return f0 * (1.0f - s) + f90 * s;
}
__device__ __forceinline__ void bwd_fresnel3(f3 f0, f3 f90, float cosTheta, f3 &d_f0, f3 &d_f90, float &d_cos, f3 d_out)
{
    float s = schlick_scale(cosTheta);
    d_f0 += d_out * (1.0f - s);
    d_f90 += d_out * s;
    if (cosTheta >= MCS_SPEC_EPS && cosTheta < 1.0f - MCS_SPEC_EPS) {
        float o = 1.0f - cosTheta, o2 = o * o;
        d_cos += sum(d_out * (f90 - f0)) * (-5.0f * (o2 * o2));
    }
}

// ---- GGX NDF (bsdf.h:76-93) -----------------------------------------------------------------
__device__ __forceinline__ float fwd_ndf_ggx(float alphaSqr, float cosTheta)
{
    xf a2 = xf(alphaSqr);
    xf c = xclamp(xf(cosTheta), xf(MCS_SPEC_EPS), xf(1.0f) - xf(MCS_SPEC_EPS));
    xf d = (c * a2 - c) * c + xf(1.0f);
    return (a2 / (d * d * xf(MCS_PI))).v;
}
__device__ __forceinline__ void bwd_ndf_ggx(float alphaSqr, float cosTheta, float &d_alphaSqr, float &d_cos, float d_out)
{
    xf a2 = xf(alphaSqr);
    xf c = xclamp(xf(cosTheta), xf(MCS_SPEC_EPS), xf(1.0f) - xf(MCS_SPEC_EPS));
    xf c2 = c * c;
    xf den = (a2 - xf(1.0f)) * c2 + xf(1.0f);
    xf den3 = den * den * den;
    d_alphaSqr += (xf(d_out) * (xf(1.0f) - (a2 + xf(1.0f)) * c2) / (xf(MCS_PI) * den3)).v;
    if (cosTheta > MCS_SPEC_EPS && cosTheta < 1.0f - MCS_SPEC_EPS)
        d_cos += (xf(d_out) * -(xf(4.0f) * (a2 - xf(1.0f)) * a2 * xf(cosTheta)) / (xf(MCS_PI) * den3)).v;
}

// ---- Smith lambda / masking (bsdf.h:98-139) --------------------------------------------------
__device__ __forceinline__ float fwd_lambda_ggx(float alphaSqr, float cosTheta)
{
    float c = clampf(cosTheta, MCS_SPEC_EPS, 1.0f - MCS_SPEC_EPS);
    float c2 = c * c;
    float t2 = (1.0f - c2) / c2;
    return 0.5f * (sqrtf(1.0f + alphaSqr * t2) - 1.0f);
}
__device__ __forceinline__ void bwd_lambda_ggx(float alphaSqr, float cosTheta, float &d_alphaSqr, float &d_cos, float d_out)
{
    float c = clampf(cosTheta, MCS_SPEC_EPS, 1.0f - MCS_SPEC_EPS);
    float c2 = c * c;
    float t2 = (1.0f - c2) / c2;
    d_alphaSqr += d_out * (0.25f * t2) * rsqrtf(alphaSqr * t2 + 1.0f);
    if (cosTheta > MCS_SPEC_EPS && cosTheta < 1.0f - MCS_SPEC_EPS)
        d_cos += d_out * -(0.5f * alphaSqr) / ((c * c2) * sqrtf(alphaSqr / c2 - alphaSqr + 1.0f));
}
__device__ __forceinline__ float fwd_masking_smith(float alphaSqr, float cosI, float cosO)
{
    return 1.0f / (1.0f + fwd_lambda_ggx(alphaSqr, cosI) + fwd_lambda_ggx(alphaSqr, cosO));
}
__device__ __forceinline__ void bwd_masking_smith(float alphaSqr, float cosI, float cosO, float &d_alphaSqr, float &d_cosI, float &d_cosO, float d_out)
{
    float s = 1.0f + fwd_lambda_ggx(alphaSqr, cosI) + fwd_lambda_ggx(alphaSqr, cosO);
    float d_l = -d_out / (s * s);
    bwd_lambda_ggx(alphaSqr, cosI, d_alphaSqr, d_cosI, d_l);
    bwd_lambda_ggx(alphaSqr, cosO, d_alphaSqr, d_cosO, d_l);
}

// ---- GGX specular lobe (bsdf.h:144-217) ------------------------------------------------------
__device__ __forceinline__ f3 fwd_pbr_specular(f3 col, f3 nrm, f3 wo, f3 wi, float alpha, float min_roughness)
{
    float woDotN = dot_exact(wo, nrm), wiDotN = dot_exact(wi, nrm);
    if (!((woDotN > MCS_SPEC_EPS) & (wiDotN > MCS_SPEC_EPS))) return F3(0.0f);
    float a = clampf(alpha, __fmul_rn(min_roughness, min_roughness), 1.0f);
    float alphaSqr = __fmul_rn(a, a);
    f3 h = safe_normalize(F3(__fadd_rn(wo.x, wi.x), __fadd_rn(wo.y, wi.y), __fadd_rn(wo.z, wi.z)));
    float woDotH = dot_exact(wo, h), nDotH = dot_exact(nrm, h);
    float D = fwd_ndf_ggx(alphaSqr, nDotH);
    float G = fwd_masking_smith(alphaSqr, woDotN, wiDotN);
    f3 F = fwd_fresnel3(col, F3(1.0f), woDotH);
    return F * (D * G * 0.25f / woDotN);
}
// Accumulates the adjoint of d_out and returns the lobe's value, fwd_pbr_specular's operations on the same intermediates (half vector,
// cosines, D, G, F and the lambda terms are evaluated once for both); callers that need only the adjoint ignore the value.
__device__ __forceinline__ f3 bwd_pbr_specular(f3 col, f3 nrm, f3 wo, f3 wi, float alpha, float min_roughness,
                                               f3 &d_col, f3 &d_nrm, f3 &d_wo, f3 &d_wi, float &d_alpha, f3 d_out)
{
    float woDotN = dot_exact(wo, nrm), wiDotN = dot_exact(wi, nrm);
    if (!((woDotN > MCS_SPEC_EPS) & (wiDotN > MCS_SPEC_EPS))) return F3(0.0f);
    float a = clampf(alpha, __fmul_rn(min_roughness, min_roughness), 1.0f);
    float alphaSqr = __fmul_rn(a, a);
    f3 hsum = F3(__fadd_rn(wo.x, wi.x), __fadd_rn(wo.y, wi.y), __fadd_rn(wo.z, wi.z));
    f3 h = safe_normalize(hsum);
    float woDotH = dot_exact(wo, h), nDotH = dot_exact(nrm, h);
    float D = fwd_ndf_ggx(alphaSqr, nDotH);
    float G = fwd_masking_smith(alphaSqr, woDotN, wiDotN);
    f3 F = fwd_fresnel3(col, F3(1.0f), woDotH);
    float k = 0.25f / woDotN;
    f3 d_F = d_out * (D * G * k);
    float dF = sum(d_out * F);
    float d_D = dF * G * k;
    float d_G = dF * D * k;
    float d_woDotN = -dF * D * G * k / woDotN;
    f3 d_f90 = F3(0.0f);
    float d_woDotH = 0.0f, d_wiDotN = 0.0f, d_nDotH = 0.0f, d_alphaSqr = 0.0f;
    bwd_fresnel3(col, F3(1.0f), woDotH, d_col, d_f90, d_woDotH, d_F);
    bwd_masking_smith(alphaSqr, woDotN, wiDotN, d_alphaSqr, d_woDotN, d_wiDotN, d_G);
    bwd_ndf_ggx(alphaSqr, nDotH, d_alphaSqr, d_nDotH, d_D);
    f3 d_h = F3(0.0f);
    bwd_dot(nrm, h, d_nrm, d_h, d_nDotH);
    bwd_dot(wo, h, d_wo, d_h, d_woDotH);
    bwd_dot(wi, nrm, d_wi, d_nrm, d_wiDotN);
    bwd_dot(wo, nrm, d_wo, d_nrm, d_woDotN);
    f3 d_hsum = F3(0.0f);
    bwd_safe_normalize(hsum, d_hsum, d_h);
    d_wo += d_hsum;
    d_wi += d_hsum;
    if (alpha > min_roughness * min_roughness) d_alpha += d_alphaSqr * 2.0f * alpha;
    return F * (D * G * 0.25f / woDotN);
}

// ---- in-kernel flavour (optixutils/c_src/bsdf.h:222-275): diffuse is a demodulated scalar ----
__device__ __forceinline__ f3 spec_color(f3 kd, f3 arm) { return (F3(0.04f * (1.0f - arm.z)) + kd * arm.z) * (1.0f - arm.x); }

__device__ __forceinline__ void ox_fwd_pbr_bsdf(f3 kd, f3 arm, f3 wo, f3 nrm, f3 wi, float min_roughness, float &diffuse, f3 &specular)
{
    diffuse = fwd_lambert(nrm, wi);
    specular = fwd_pbr_specular(spec_color(kd, arm), nrm, wo, wi, __fmul_rn(arm.y, arm.y), min_roughness);
}
// Value and adjoint in one pass, for the backward passes, which need both (the value weights the light gradient): diffuse / specular
// are ox_fwd_pbr_bsdf's value, with the FMAs of the Lambert dot product spelled out so that it rounds the same wherever the body is
// inlined (the lobe's one FMA, in Fresnel, has no other way to contract), and the adjoints of d_diffuse / d_specular are accumulated
// into d_kd, d_arm, d_wo, d_nrm.
// diffuse_only: Lambert alone (BSDF 'diffuse' and 'white'), which has no kd, arm or wo adjoint.
// d_wo is returned so the caller can push it through wo = normalize(view_pos - pos) once per pixel
// (the map is linear in d_wo, so summing d_wo over samples first is exact up to rounding).
__device__ __forceinline__ void ox_fwdbwd_pbr_bsdf(bool diffuse_only, f3 kd, f3 arm, f3 wo, f3 nrm, f3 wi, float min_roughness, float d_diffuse,
                                                   f3 d_specular, float &diffuse, f3 &specular, f3 &d_kd, f3 &d_arm, f3 &d_wo, f3 &d_nrm)
{
    const float nDotWi = __fmaf_rn(nrm.z, wi.z, __fmaf_rn(nrm.x, wi.x, __fmul_rn(nrm.y, wi.y)));     // dot(nrm, wi) as fwd_lambert contracts it
    diffuse = fmaxf(nDotWi * MCS_INV_PI, 0.0f);
    specular = F3(0.0f);
    float d_alpha = 0.0f;
    f3 d_sc = F3(0.0f), d_wi = F3(0.0f);
    if (!diffuse_only)
        specular = bwd_pbr_specular(spec_color(kd, arm), nrm, wo, wi, __fmul_rn(arm.y, arm.y), min_roughness, d_sc, d_nrm, d_wo, d_wi, d_alpha, d_specular);
    if (nDotWi > 0.0f) bwd_dot(nrm, wi, d_nrm, d_wi, d_diffuse * MCS_INV_PI);                        // bwd_lambert
    if (diffuse_only) return;
    d_kd -= d_sc * ((arm.x - 1.0f) * arm.z);
    d_arm.x += sum(d_sc * ((F3(0.04f) - kd) * arm.z - F3(0.04f)));
    d_arm.z -= sum(d_sc * (kd - F3(0.04f))) * (arm.x - 1.0f);
    d_arm.y += d_alpha * 2.0f * arm.y;
}

// ---- Frostbite diffuse (renderutils/c_src/bsdf.cu:72-153) -------------------------------------
__device__ __forceinline__ float fwd_frostbite(f3 nrm, f3 wi, f3 wo, float lr)
{
    float wiDotN = dot(wi, nrm), woDotN = dot(wo, nrm);
    if (!(wiDotN > 0.0f && woDotN > 0.0f)) return 0.0f;
    f3 h = safe_normalize(wo + wi);
    float wiDotH = dot(wi, h);
    float energyBias = 0.5f * lr;
    float energyFactor = 1.0f - (0.51f / 1.51f) * lr;
    float f90 = energyBias + 2.0f * wiDotH * wiDotH * lr;
    return fwd_fresnel1(1.0f, f90, wiDotN) * fwd_fresnel1(1.0f, f90, woDotN) * energyFactor;
}
__device__ __forceinline__ void bwd_frostbite(f3 nrm, f3 wi, f3 wo, float lr, f3 &d_nrm, f3 &d_wi, f3 &d_wo, float &d_lr, float d_out)
{
    float wiDotN = dot(wi, nrm), woDotN = dot(wo, nrm);
    if (!(wiDotN > 0.0f && woDotN > 0.0f)) return;
    f3 hsum = wo + wi;
    f3 h = safe_normalize(hsum);
    float wiDotH = dot(wi, h);
    float energyBias = 0.5f * lr;
    float energyFactor = 1.0f - (0.51f / 1.51f) * lr;
    float f90 = energyBias + 2.0f * wiDotH * wiDotH * lr;
    float wiS = fwd_fresnel1(1.0f, f90, wiDotN), woS = fwd_fresnel1(1.0f, f90, woDotN);
    float d_wiS = d_out * woS * energyFactor, d_woS = d_out * wiS * energyFactor, d_ef = d_out * wiS * woS;
    float d_woDotN = 0.0f, d_wiDotN = 0.0f, d_f0 = 0.0f, d_f90 = 0.0f;
    bwd_fresnel1(1.0f, f90, woDotN, d_f0, d_f90, d_woDotN, d_woS);
    bwd_fresnel1(1.0f, f90, wiDotN, d_f0, d_f90, d_wiDotN, d_wiS);
    float d_wiDotH = d_f90 * 4.0f * wiDotH * lr;
    d_lr += d_f90 * 2.0f * wiDotH * wiDotH;
    d_lr -= (0.51f / 1.51f) * d_ef;
    d_lr += 0.5f * d_f90;
    f3 d_h = F3(0.0f);
    bwd_dot(wi, h, d_wi, d_h, d_wiDotH);
    f3 d_hsum = F3(0.0f);
    bwd_safe_normalize(hsum, d_hsum, d_h);
    d_wi += d_hsum; d_wo += d_hsum;
    bwd_dot(wo, nrm, d_wo, d_nrm, d_woDotN);
    bwd_dot(wi, nrm, d_wi, d_nrm, d_wiDotN);
}

// ---- stand-alone flavour (renderutils/c_src/bsdf.cu:300-377): kd-modulated diffuse ------------
__device__ __forceinline__ f3 ru_fwd_pbr_bsdf(f3 kd, f3 arm, f3 pos, f3 nrm, f3 view_pos, f3 light_pos, float min_roughness, int BSDF)
{
    f3 wo = safe_normalize(view_pos - pos), wi = safe_normalize(light_pos - pos);
    float diff = BSDF == 0 ? fwd_lambert(nrm, wi) : fwd_frostbite(nrm, wi, wo, arm.y);
    f3 diffuse = kd * ((1.0f - arm.z) * diff);
    return diffuse + fwd_pbr_specular(spec_color(kd, arm), nrm, wo, wi, __fmul_rn(arm.y, arm.y), min_roughness);
}
__device__ __forceinline__ void ru_bwd_pbr_bsdf(f3 kd, f3 arm, f3 pos, f3 nrm, f3 view_pos, f3 light_pos, float min_roughness, int BSDF,
                                                f3 &d_kd, f3 &d_arm, f3 &d_pos, f3 &d_nrm, f3 &d_view_pos, f3 &d_light_pos, f3 d_out)
{
    f3 _wi = light_pos - pos, _wo = view_pos - pos;
    f3 wi = safe_normalize(_wi), wo = safe_normalize(_wo);
    f3 sc = spec_color(kd, arm);
    f3 diff_col = kd * (1.0f - arm.z);
    float diff = BSDF == 0 ? fwd_lambert(nrm, wi) : fwd_frostbite(nrm, wi, wo, arm.y);
    float d_alpha = 0.0f;
    f3 d_sc = F3(0.0f), d_wi = F3(0.0f), d_wo = F3(0.0f);
    bwd_pbr_specular(sc, nrm, wo, wi, __fmul_rn(arm.y, arm.y), min_roughness, d_sc, d_nrm, d_wo, d_wi, d_alpha, d_out);
    float d_diff = sum(diff_col * d_out);
    if (BSDF == 0) bwd_lambert(nrm, wi, d_nrm, d_wi, d_diff);
    else bwd_frostbite(nrm, wi, wo, arm.y, d_nrm, d_wi, d_wo, d_arm.y, d_diff);
    f3 d_diff_col = d_out * diff;
    d_kd += d_diff_col * (1.0f - arm.z);
    d_arm.z -= sum(d_diff_col * kd);
    d_kd -= d_sc * ((arm.x - 1.0f) * arm.z);
    d_arm.x += sum(d_sc * ((F3(0.04f) - kd) * arm.z - F3(0.04f)));
    d_arm.z -= sum(d_sc * (kd - F3(0.04f))) * (arm.x - 1.0f);
    d_arm.y += d_alpha * 2.0f * arm.y;
    f3 d__wi = F3(0.0f);
    bwd_safe_normalize(_wi, d__wi, d_wi);
    d_light_pos += d__wi; d_pos -= d__wi;
    f3 d__wo = F3(0.0f);
    bwd_safe_normalize(_wo, d__wo, d_wo);
    d_view_pos += d__wo; d_pos -= d__wo;
}

// ---- shading normal (renderutils/c_src/normal.cu:17-90) ---------------------------------------
#define MCS_NORMAL_THRESHOLD 0.1f
__device__ __forceinline__ f3 fwd_perturb_normal(f3 pn, f3 sn, f3 st, bool opengl)
{
    f3 bit = safe_normalize(cross(st, sn));
    float sg = opengl ? -1.0f : 1.0f;
    return safe_normalize(st * pn.x + bit * (sg * pn.y) + sn * fmaxf(pn.z, 0.0f));
}
__device__ __forceinline__ void bwd_perturb_normal(f3 pn, f3 sn, f3 st, f3 &d_pn, f3 &d_sn, f3 &d_st, f3 d_out, bool opengl)
{
    f3 _bit = cross(st, sn);
    f3 bit = safe_normalize(_bit);
    float sg = opengl ? -1.0f : 1.0f;
    f3 _s = st * pn.x + bit * (sg * pn.y) + sn * fmaxf(pn.z, 0.0f);
    f3 d_s = F3(0.0f);
    bwd_safe_normalize(_s, d_s, d_out);
    if (pn.z > 0.0f) { d_sn += d_s * pn.z; d_pn.z += sum(d_s * sn); }
    f3 d_bit = d_s * (sg * pn.y);
    d_pn.y += sg * sum(d_s * bit);
    d_st += d_s * pn.x;
    d_pn.x += sum(d_s * st);
    f3 d__bit = F3(0.0f);
    bwd_safe_normalize(_bit, d__bit, d_bit);
    bwd_cross(st, sn, d_st, d_sn, d__bit);
}
__device__ __forceinline__ f3 fwd_bend_normal(f3 view_vec, f3 sn, f3 gn)
{
    float t = clampf(dot(view_vec, sn) / MCS_NORMAL_THRESHOLD, 0.0f, 1.0f);
    return gn * (1.0f - t) + sn * t;
}
__device__ __forceinline__ void bwd_bend_normal(f3 view_vec, f3 sn, f3 gn, f3 &d_view, f3 &d_sn, f3 &d_gn, f3 d_out)
{
    float dp = dot(view_vec, sn);
    float t = clampf(dp / MCS_NORMAL_THRESHOLD, 0.0f, 1.0f);
    if (dp > MCS_NORMAL_THRESHOLD) d_sn += d_out;
    else {
        d_gn += d_out * (1.0f - t);
        d_sn += d_out * t;
        float d_t = sum(d_out * (sn - gn));
        float d_dp = (dp < 0.0f || dp > MCS_NORMAL_THRESHOLD) ? 0.0f : d_t / MCS_NORMAL_THRESHOLD;
        bwd_dot(view_vec, sn, d_view, d_sn, d_dp);
    }
}
