// Driver of the packing core (medaka_b200/csrc/packing.h) with a fake engine, for tests/test_packing.py.  Commands on
// stdin, one per line:
//   gmax G       windows per group (default 1 << 30)
//   cap C        windows the fake buffers hold (default unlimited)
//   call B L     one call of B windows of length L, with a ticket
//   alone B L    the one-call form: launch the open group, then the call with a group limit of max(B, G)
//   wait K       settle ticket K
//   flush        launch the open group
// and the engine's operations and the core's answers on stdout:
//   open W | stage CALL FIRST N AT | launch SERIAL LEN WINDOWS CALL:FIRST+N ... | ticket K | wait K GROUP
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>

#include "../../medaka_b200/csrc/packing.h"

using mdk::Packing;

static float tags[1 << 16];   // call i's probabilities "buffer" is tags + i: the pieces name their call by it

struct Fake {
    Packing *pk;
    int64_t cap = INT64_MAX;
    int call = -1;

    int open(int64_t windows) { printf("open %lld\n", (long long)windows); return 0; }
    int64_t capacity(int64_t) { return cap; }
    int stage(int64_t first, int64_t n, int64_t at) {
        printf("stage %d %lld %lld %lld\n", call, (long long)first, (long long)n, (long long)at);
        return 0;
    }
    int launch() {
        printf("launch %lld %lld %lld", (long long)pk->serial, (long long)pk->len, (long long)pk->windows);
        for (const Packing::Piece &p : pk->pieces)
            printf(" %d:%lld+%lld", (int)(p.probs - tags), (long long)p.first, (long long)p.n);
        printf("\n");
        return 0;
    }
};

int main() {
    static Packing pk;
    Fake eng{&pk};
    int64_t gmax = 1 << 30;
    std::string cmd;
    while (std::cin >> cmd) {
        int64_t a = 0, b = 0, ticket = -1, group = -1;
        int rc = 0;
        if (cmd == "gmax") {
            std::cin >> gmax;
        } else if (cmd == "cap") {
            std::cin >> eng.cap;
        } else if (cmd == "call" || cmd == "alone") {
            std::cin >> a >> b;
            eng.call++;
            int64_t g = gmax;
            if (cmd == "alone") {
                rc = pk.launch(eng);
                g = std::max(a, gmax);
            }
            if (!rc) rc = pk.enqueue(eng, a, b, tags + eng.call, nullptr, nullptr, g, &ticket);
            if (!rc) printf("ticket %lld\n", (long long)ticket);
        } else if (cmd == "wait") {
            std::cin >> a;
            rc = pk.settle(eng, a, &group);
            if (!rc) printf("wait %lld %lld\n", (long long)a, (long long)group);
        } else if (cmd == "flush") {
            rc = pk.launch(eng);
        } else {
            fprintf(stderr, "unknown command %s\n", cmd.c_str());
            return 2;
        }
        if (rc) return 1;
    }
    return 0;
}
