// emul.cu -- runs the per-thread phases of fftcore.cuh thread-by-thread on the CPU and compares with a float64 DFT.
//   nvcc -O2 -std=c++17 -I passiveradar_b200/csrc -o /tmp/fft_emul scripts/fft/emul.cu && /tmp/fft_emul
//   /tmp/fft_emul seeds      frame_pass_kernel's twiddle source (Tw1Seeds, R3 = 8) against the table: one key=value line
// No CUDA runtime call is made: this pins the index algebra / twiddle conventions without a GPU.
#include <cmath>
#include <complex>
#include <cstdio>
#include <random>
#include <string>
#include <vector>
#include "fftcore.cuh"

using namespace prc::fft;
typedef std::complex<double> cd;

template <int R3>
void make_tw(std::vector<float2>& tw) {
    using G = Geo<R3>;
    tw.resize(G::TW1 + G::TW2);
    for (int i = 0; i < G::TW1; ++i) {
        const int k1 = i / G::T, t = i % G::T;
        const double a = -2.0 * M_PI * (double)((long long)t * k1 % G::L) / G::L;
        tw[i] = make_float2((float)cos(a), (float)sin(a));
    }
    for (int q = 0; q < G::TW2; ++q) {
        const int k2 = q / R3, n3 = q % R3;
        const double a = -2.0 * M_PI * (double)(n3 * k2) / (16 * R3);
        tw[G::TW1 + q] = make_float2((float)cos(a), (float)sin(a));
    }
}

template <int R3>
int run() {
    using G = Geo<R3>;
    std::mt19937 rng(1234 + R3);
    std::normal_distribution<float> nd;
    std::vector<float2> x(G::L), tw;
    for (auto& v : x) v = make_float2(nd(rng), nd(rng));
    make_tw<R3>(tw);
    const float2* tw1 = tw.data();
    const float2* tw2 = tw.data() + G::TW1;
    std::vector<float2> ea(G::EX), eb(G::EX);
    struct Regs { float2 v[16]; };
    std::vector<Regs> regs(G::T);
    // float64 DFT
    std::vector<cd> X(G::L);
    for (int k = 0; k < G::L; ++k) {
        cd s = 0;
        for (int n = 0; n < G::L; ++n) {
            const double a = -2.0 * M_PI * (double)((long long)n * k % G::L) / G::L;
            s += cd(x[n].x, x[n].y) * cd(cos(a), sin(a));
        }
        X[k] = s;
    }
    double xmax = 0;
    for (auto& v : X) xmax = std::max(xmax, std::abs(v));
    // n2p
    for (int t = 0; t < G::T; ++t) for (int n1 = 0; n1 < 16; ++n1) regs[t].v[n1] = x[n1 * G::T + t];
    for (int t = 0; t < G::T; ++t) n2p_pass1<R3>(regs[t].v, t, ea.data(), Tw1Table<R3>{tw1});
    for (int t = 0; t < G::T; ++t) n2p_pass2<R3>(regs[t].v, t, ea.data(), eb.data(), tw2);
    for (int t = 0; t < G::T; ++t) n2p_pass3<R3>(regs[t].v, t, eb.data());
    double e1 = 0;
    std::vector<int> seen(G::L, 0);
    for (int t = 0; t < G::T; ++t)
        for (int r = 0; r < 16; ++r) {
            const int f = perm_freq<R3>(t, r);
            seen[f]++;
            e1 = std::max(e1, std::abs(cd(regs[t].v[r].x, regs[t].v[r].y) - X[f]));
        }
    int bad = 0;
    for (int f = 0; f < G::L; ++f) bad += seen[f] != 1;
    // p2n applied to the permuted spectrum: y[n] = sum_k X[k] W^{nk}  ==  L * x[(-n) mod L]
    for (int t = 0; t < G::T; ++t) p2n_pass1<R3>(regs[t].v, t, eb.data());
    for (int t = 0; t < G::T; ++t) p2n_pass2<R3>(regs[t].v, t, eb.data(), ea.data(), tw2);
    for (int t = 0; t < G::T; ++t) p2n_pass3<R3>(regs[t].v, t, ea.data(), Tw1Table<R3>{tw1});
    double e2 = 0, ymax = 0;
    for (int t = 0; t < G::T; ++t)
        for (int n1 = 0; n1 < 16; ++n1) {
            const int n = n1 * G::T + t;
            const float2 want = x[(G::L - n) % G::L];
            const cd w((double)want.x * G::L, (double)want.y * G::L);
            ymax = std::max(ymax, std::abs(w));
            e2 = std::max(e2, std::abs(cd(regs[t].v[n1].x, regs[t].v[n1].y) - w));
        }
    printf("R3=%2d L=%4d: n2p err %.3e (rel %.2e), perm bijective: %s, p2n(n2p(x)) err rel %.2e\n", R3, G::L, e1, e1 / xmax,
           bad ? "NO" : "yes", e2 / ymax);
    return (e1 / xmax < 2e-6 && !bad && e2 / ymax < 4e-6) ? 0 : 1;
}

// Largest error of n2p (x -> X, relative to max |X|) and of p2n alone (permuted z -> y[n] = sum_k z[k] W^{nk}, relative
// to max |y|) over `trials` random inputs, with the pass-1 / pass-3 twiddles of thread t from src(t).
template <int R3, class Src>
void source_errors(const std::vector<float2>& tw, Src src, int trials, double& en2p, double& ep2n) {
    using G = Geo<R3>;
    const float2* tw2 = tw.data() + G::TW1;
    std::vector<float2> ea(G::EX), eb(G::EX), x(G::L);
    struct Regs { float2 v[16]; };
    std::vector<Regs> regs(G::T);
    std::vector<cd> W(G::L);
    for (int m = 0; m < G::L; ++m) W[m] = std::polar(1.0, -2.0 * M_PI * m / G::L);
    auto dft = [&](const std::vector<float2>& in, std::vector<cd>& out) {
        out.assign(G::L, 0);
        for (int k = 0; k < G::L; ++k)
            for (int n = 0; n < G::L; ++n) out[k] += cd(in[n].x, in[n].y) * W[(long long)n * k % G::L];
    };
    std::mt19937 rng(4321 + R3);
    std::normal_distribution<float> nd;
    std::vector<cd> X;
    en2p = ep2n = 0;
    for (int trial = 0; trial < trials; ++trial) {
        for (auto& v : x) v = make_float2(nd(rng), nd(rng));
        dft(x, X);
        for (int t = 0; t < G::T; ++t) for (int n1 = 0; n1 < 16; ++n1) regs[t].v[n1] = x[n1 * G::T + t];
        for (int t = 0; t < G::T; ++t) n2p_pass1<R3>(regs[t].v, t, ea.data(), src(t));
        for (int t = 0; t < G::T; ++t) n2p_pass2<R3>(regs[t].v, t, ea.data(), eb.data(), tw2);
        for (int t = 0; t < G::T; ++t) n2p_pass3<R3>(regs[t].v, t, eb.data());
        double e = 0, xmax = 0;
        for (auto& v : X) xmax = std::max(xmax, std::abs(v));
        for (int t = 0; t < G::T; ++t)
            for (int r = 0; r < 16; ++r) e = std::max(e, std::abs(cd(regs[t].v[r].x, regs[t].v[r].y) - X[perm_freq<R3>(t, r)]));
        en2p = std::max(en2p, e / xmax);
        // p2n of x laid out in permuted order: register r of thread t holds z[perm_freq(t, r)] = x[perm_freq(t, r)]
        for (int t = 0; t < G::T; ++t) for (int r = 0; r < 16; ++r) regs[t].v[r] = x[perm_freq<R3>(t, r)];
        for (int t = 0; t < G::T; ++t) p2n_pass1<R3>(regs[t].v, t, eb.data());
        for (int t = 0; t < G::T; ++t) p2n_pass2<R3>(regs[t].v, t, eb.data(), ea.data(), tw2);
        for (int t = 0; t < G::T; ++t) p2n_pass3<R3>(regs[t].v, t, ea.data(), src(t));
        e = 0;                                   // y = DFT(x): the DFT matrix is symmetric, so X is the wanted output
        for (int t = 0; t < G::T; ++t)
            for (int n1 = 0; n1 < 16; ++n1) e = std::max(e, std::abs(cd(regs[t].v[n1].x, regs[t].v[n1].y) - X[n1 * G::T + t]));
        ep2n = std::max(ep2n, e / xmax);
    }
}

// Tw1Seeds<8> (frame_pass_kernel's pass-1 / pass-3 twiddles) against float64 and, through whole transforms, against
// the table it replaces
int seeds() {
    constexpr int R3 = 8;
    using G = Geo<R3>;
    std::vector<float2> tw;
    make_tw<R3>(tw);
    const float2* tw1 = tw.data();
    double ulp = 0;                              // largest component error of a twiddle, in units of 2^-23 (1 ulp of 1.0)
    for (int t = 0; t < G::T; ++t) {
        const Tw1Seeds<R3> s(tw1, t);
        for (int k1 = 1; k1 < 16; ++k1) {
            const float2 w = s(t, k1);
            const double a = -2.0 * M_PI * (double)((long long)t * k1 % G::L) / G::L;
            ulp = std::max(ulp, std::max(std::abs(w.x - cos(a)), std::abs(w.y - sin(a))) * 8388608.0);
        }
    }
    double tn, tp, sn, sp;
    source_errors<R3>(tw, [&](int) { return Tw1Table<R3>{tw1}; }, 4, tn, tp);
    source_errors<R3>(tw, [&](int t) { return Tw1Seeds<R3>(tw1, t); }, 4, sn, sp);
    printf("twiddle_ulp=%.4f table_n2p=%.4e seeded_n2p=%.4e table_p2n=%.4e seeded_p2n=%.4e smem_seeded_float2=%d "
           "smem_table_float2=%d\n", ulp, tn, sn, tp, sp, SmemSeeded<R3>::SMEM_FLOAT2, G::SMEM_FLOAT2);
    return 0;
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "seeds") return seeds();
    int rc = run<4>() | run<8>() | run<16>();
    printf(rc ? "FAIL\n" : "OK\n");
    return rc;
}
