# ORACLE build (test infrastructure): the campaign oracle.  Output: oracle/liboracle_campaign.so (git-ignored).
# The same sources as liboracle.so (Makefile) plus campaign.c: the Fuzzer restated in C and oracle_fuzz_campaign.
CC ?= gcc
CFLAGS ?= -O3 -march=native -fPIC -Wall -Wextra -std=gnu11 -pthread
SRCS := machine.c models.c model_ir.c fuzz.c ddmin.c sts.c dpor.c dpor_frontier.c intmin.c provenance.c campaign.c
liboracle_campaign.so: $(SRCS) machine.h jrandom.h ../include/demi_b200.h ../include/demi_limits.h ../include/demi_model_ir.h
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS)
clean:
	rm -f liboracle_campaign.so
