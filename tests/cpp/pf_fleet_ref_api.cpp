// A fleet of particle filters written against include/crb/reference_api.hpp: seven robots, each at its own pose with
// its own control, observe the demo's RFID tags within MAX_RANGE (src/particle_filter.cpp:192-196, :257-268) and run
// the demo's tick, pf_localization + resampling (:270-271), through the fleet overload.  Robot r's generators are
// seeded with 100 + r and 200 + r.  The program prints its inputs, the draws the reference's loops would make with
// those generators (two normals per particle, then one uniform per particle), its outputs as hex floats, and a
// checksum, so that a checker can recompute the tick.
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "crb/reference_api.hpp"

constexpr int NP = 100;

static void put(const char* name, const float* v, size_t n) {
  std::printf("%s", name);
  for (size_t i = 0; i < n; ++i) std::printf(" %a", (double)v[i]);
  std::printf("\n");
}

int main() {
  const int nr = 7;
  const float PI = 3.141592653f, MAX_RANGE = 20.0f, Qsim = 0.04f;
  const float rfid[4][2] = {{10.0f, 0.0f}, {10.0f, 10.0f}, {0.0f, 15.0f}, {-5.0f, 20.0f}};
  crb::Matrix2f Rsim = crb::Matrix2f::Identity();
  Rsim(0, 0) = 1.0f * 1.0f;
  Rsim(1, 1) = 30.0f / 180.0f * PI * 30.0f / 180.0f * PI;
  const float Q = 0.01f;
  std::vector<crb::Mat<4, NP>> px(nr);
  std::vector<crb::Mat<NP, 1>> pw(nr);
  std::vector<crb::Vector4f> xEst;
  std::vector<crb::Matrix4f> PEst;
  std::vector<std::vector<crb::RowVector3f>> z(nr);
  std::vector<crb::Vector2f> u(nr);
  std::vector<std::mt19937> gen, gen2;
  std::normal_distribution<> gaussian_d{0, 1};
  std::uniform_real_distribution<> uni_d{1.0, 2.0};
  std::mt19937 scene(7);
  std::uniform_real_distribution<> pose(-8.0, 8.0), yaw(-PI, PI);
  for (int r = 0; r < nr; ++r) {
    gen.emplace_back(100 + r);
    gen2.emplace_back(200 + r);
    const float tx = (float)pose(scene), ty = (float)pose(scene);
    for (int ip = 0; ip < NP; ++ip) {
      px[r](0, ip) = tx + 0.2f * (float)gaussian_d(scene);
      px[r](1, ip) = ty + 0.2f * (float)gaussian_d(scene);
      px[r](2, ip) = (float)yaw(scene);
      px[r](3, ip) = 1.0f;
      pw[r](ip) = 1.0f / NP;
    }
    u[r](0) = 0.5f + 0.1f * (float)r;
    u[r](1) = 0.1f - 0.03f * (float)r;
    for (int i = 0; i < 4; ++i) {
      const float dx = tx - rfid[i][0], dy = ty - rfid[i][1];
      const float d = std::sqrt(dx * dx + dy * dy);
      if (d <= MAX_RANGE) {
        crb::RowVector3f zi;
        zi(0, 0) = d + (float)gaussian_d(scene) * Qsim;
        zi(0, 1) = rfid[i][0];
        zi(0, 2) = rfid[i][1];
        z[r].push_back(zi);
      }
    }
  }
  std::printf("nr %d np %d\n", nr, NP);
  for (int r = 0; r < nr; ++r) {
    put("px", px[r].data(), 4 * NP);   // Eigen layout: particle-major
    put("pw", pw[r].data(), NP);
    put("u", u[r].data(), 2);
    std::vector<float> zr;
    for (const auto& zi : z[r])
      for (int k = 0; k < 3; ++k) zr.push_back(zi(0, k));
    put("z", zr.data(), zr.size());
    std::mt19937 g = gen[r], g2 = gen2[r];   // what the reference's loops draw with copies of the generators
    std::normal_distribution<> gd = gaussian_d;
    std::uniform_real_distribution<> ud = uni_d;
    std::vector<float> nz(2 * NP), un(NP);
    for (int ip = 0; ip < NP; ++ip) {
      nz[ip] = (float)gd(g);
      nz[NP + ip] = (float)gd(g);
    }
    for (int ip = 0; ip < NP; ++ip) un[ip] = (float)ud(g2);
    put("noise", nz.data(), nz.size());
    put("uniforms", un.data(), un.size());
  }
  pf_localization_resampling<NP>(px, pw, xEst, PEst, z, u, Rsim, Q, gen, gaussian_d, gen2, uni_d);
  double checksum = 0.0;
  for (int r = 0; r < nr; ++r) {
    put("px_out", px[r].data(), 4 * NP);
    put("pw_out", pw[r].data(), NP);
    put("xEst", xEst[r].data(), 4);
    put("PEst", PEst[r].data(), 16);
    for (int k = 0; k < 4; ++k) checksum += xEst[r](k);
  }
  std::printf("checksum %.9e\n", checksum);
  return 0;
}
