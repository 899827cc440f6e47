// Host build of sample_parts.hpp (how a read or pair sketch is cut into hash-range parts within a device memory budget).
//
// stdin, one case per line: "bases records mates k c grouped budget fixed forced".  stdout, one line per case:
//   "ok thr nbk Mb need P" followed by P lines "lo hi g0 ng events bytes",
//   or "events" (more than 2^32-2 events per part even at the most parts) or "oom need".
#include <cstdint>
#include <iostream>
#include <sstream>
#include <string>

#include "sample_parts.hpp"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        uint64_t bases = 0, records = 0, c = 1, budget = 0, fixed = 0;
        int mates = 1, k = 31, grouped = 1;
        uint32_t forced = 0;
        in >> bases >> records >> mates >> k >> c >> grouped >> budget >> fixed >> forced;
        syl::SamplePlan plan;
        const int rc = syl::plan_sample_parts(bases, records, mates, k, c, grouped != 0, budget, fixed, forced, plan);
        if (rc == syl::PLAN_TOO_MANY_EVENTS) { std::cout << "events\n"; continue; }
        if (rc == syl::PLAN_OVER_BUDGET) { std::cout << "oom " << plan.need << "\n"; continue; }
        std::cout << "ok " << plan.map.thr << " " << plan.map.nbk << " " << plan.map.Mb << " " << plan.need << " "
                  << plan.parts.size() << "\n";
        for (const syl::SamplePart &p : plan.parts)
            std::cout << p.lo << " " << p.hi << " " << p.g0 << " " << p.ng << " " << p.events << " " << p.bytes << "\n";
    }
    return 0;
}
