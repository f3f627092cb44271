// Prints the launch plan of csrc/fps_plan.h for every query line on stdin (tests/test_fps_plan_cpu.py):
//   fps n c m cluster flags aligned  |  dist n cluster  |  features n c cluster
// -> kind cl p cp smem temp(full range) temp(partial range) rounds
// A route whose full range does not run partial ranges may send them to another kernel (the F-FPS bucket route); its
// line then ends with that partial-range plan: kind cl p cp smem.
#include <cstdio>
#include <iostream>
#include <string>

#include "../3dssd_b200/csrc/fps_plan.h"

using namespace ssd3d;

static const char *kind_name(FpsKind k)
{
    switch (k) {
    case FpsKind::Bucket: return "bucket";
    case FpsKind::Direct: return "direct";
    case FpsKind::Packet: return "packet";
    case FpsKind::Generic: return "generic";
    case FpsKind::Dist: return "dist";
    case FpsKind::Features: return "features";
    case FpsKind::FeaturesBucket: return "features_bucket";
    case FpsKind::Fallback: return "fallback";
    }
    return "?";
}

int main()
{
    std::string fam;
    while (std::cin >> fam) {
        FpsPlan full, part;
        if (fam == "fps") {
            int n, c, m, cluster, flags, aligned;
            std::cin >> n >> c >> m >> cluster >> flags >> aligned;
            full = plan_fps(n, c, m, cluster, flags, aligned != 0, (long long)n * c, false);
            part = plan_fps(n, c, m, cluster, flags, aligned != 0, (long long)n * c, true);
        } else if (fam == "dist") {
            int n, cluster;
            std::cin >> n >> cluster;
            full = part = plan_fps_dist(n, cluster);
        } else {
            int n, c, cluster;
            std::cin >> n >> c >> cluster;
            full = plan_ffps(n, c, cluster, false);
            part = plan_ffps(n, c, cluster, true);
        }
        const bool same = full.kind == part.kind && full.cl == part.cl && full.p == part.p && full.smem == part.smem;
        if (!same && (full.rounds || full.kind == part.kind)) return 1;
        std::printf("%s %d %d %d %zu %ld %ld %d", kind_name(full.kind), full.cl, full.p, full.cp, full.smem, full.temp,
                    part.temp, (int)full.rounds);
        if (!same) std::printf(" %s %d %d %d %zu", kind_name(part.kind), part.cl, part.p, part.cp, part.smem);
        std::printf("\n");
    }
    return 0;
}
