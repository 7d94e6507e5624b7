# Builds the zone-monitoring oracle (orc_zone.c) on its own; same flags as oracle/Makefile (the reference's
# Release defaults, -ffp-contract=off pins "no FMA").  Test infrastructure only.
CC := /usr/bin/gcc
CFLAGS = -O3 -DNDEBUG -std=c11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

all: libouster_oracle_zone.so

libouster_oracle_zone.so: orc_zone.c
	$(CC) $(CFLAGS) -shared -o $@ orc_zone.c -lm

clean:
	rm -f libouster_oracle_zone.so
